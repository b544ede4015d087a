/*
 * traceweaver_b200.h — C ABI of the B200-native span-assignment engine.
 *
 * Drop-in scope: ONE path of Sachin-A/TraceWeaver — `TraceWeaverV3.FindAssignments` for
 * method "MaxScoreBatchSubsetWithSkips" (reference
 * src/trace_reconstructor/ports/python/algorithms/traceweaver_v3.py:1087-1229, called from
 * executor.py:1172-1175).  The reference has no FFI of its own (it is single-process Python, its
 * C++ "port" is an empty skeleton — ports/cpp/scheme.cpp:8-10), so the entry points below are
 * what a ctypes binding placed inside `TraceWeaverV3.FindAssignments` would call; INTEGRATION.md
 * shows that stub.  Every entry point names the reference code it replaces.
 *
 * Conventions
 *   - plain C, no torch / C++ types in any signature; all buffers are caller-owned.
 *   - every pointer inside tw_batch / tw_params / tw_pass_out is a DEVICE pointer unless the
 *     field comment says "host".  `stream` is a cudaStream_t passed as void*.
 *   - every function returns TW_OK (0) or a negative tw_status; nothing throws across the ABI.
 *   - times are int64 microseconds (Jaeger startTime is ~1.7e15 us: differences are formed in
 *     int64 BEFORE conversion to double); scores are IEEE double.  Fractional (float64) microseconds
 *     enter through tw_engine_bind_f64, which moves them into exact int64 fixed point.
 *   - "problem" = one service: one incoming endpoint with n_in spans and E outgoing endpoints
 *     ("eps") in the topological order of the invocation graph (traceweaver_v1.py:37-39).
 *     In-spans and each ep's out-spans are sorted by (start, end) (executor.py:1111-1112).
 *     A batch concatenates many problems so one launch sequence covers all of them.
 */
#ifndef TRACEWEAVER_B200_H
#define TRACEWEAVER_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TW_ABI_VERSION 6

/* Algorithm constants hard-coded by the reference. */
#define TW_MAX_E 8             /* engine limit on out-eps per service (shipped data: <= 4)      */
#define TW_K 5                 /* topK                    traceweaver_v3.py:1109                */
#define TW_MAX_WINDOW 30       /* batch_size_mis          traceweaver_v3.py:1108                */
#define TW_WINDOW_CAP 31       /* a window opened by a perfect cut can reach 31 (v3:1063-1072) */
#define TW_PARAM_BATCH 100     /* batch_size              traceweaver_v3.py:1107                */
#define TW_PARAM_NBATCHES 10   /* nbatches                traceweaver_v3.py:599                 */
#define TW_WEIGHT_OFFSET 10000.0 /* MWIS vertex weight    traceweaver_v3.py:1260                */
/* Independent sets whose total weights differ by less than this are TIED.  The reference hands the
 * instance to Gurobi (traceweaver_v3.py:1411), which returns an arbitrary optimum on ties; the engine
 * and the oracle both return, per connected component of the window's conflict graph, the FIRST tied
 * optimum in depth-first order (in-spans ascending; ranks ascending, "unassigned" last).  The
 * tolerance makes that choice independent of the order in which a solver adds the weights up. */
#define TW_MWIS_TIE_TOL 1e-6
#define TW_GMM_MAX_COMP 5      /* max mixture components  traceweaver_v3.py:768                 */
#define TW_GAUSS_REC 3         /* doubles per pass-0 record: mu, sigma, log(sigma)              */
#define TW_MIX_REC 21          /* doubles per mixture record: k, pc[5], mu*pc[5], logdet[5], logw[5] */

typedef enum tw_status {
  TW_OK = 0,
  TW_ERR_INVALID = -1,        /* malformed descriptor (E > TW_MAX_E, empty problem, bad offsets) */
  TW_ERR_CUDA = -2,           /* a CUDA runtime call failed; see tw_last_error()                 */
  TW_ERR_MWIS_LIMIT = -3,     /* exact MWIS branch-and-bound exceeded its node budget            */
  TW_ERR_RANGE_LIMIT = -4,    /* an in-span has more candidates per ep than the engine supports  */
  TW_ERR_UNSUPPORTED = -5,    /* skip budgets != 0 (n_out != n_in) handed to the two-pass entry points:
                                 such services go through tw_skip_solve                            */
  TW_ERR_NO_DEVICE = -6,      /* no CUDA device / wrong architecture                              */
  TW_ERR_REFERENCE_UNDEFINED = -7 /* skip mode: the reference itself raises on this input (two tuples
                                 with equal scores that differ in a skip span, an all-skip tuple, a
                                 chain of skipped ancestors, a missing distribution key)          */
} tw_status;

/* Term kinds of the score (traceweaver_v1.py:316-357). */
#define TW_TERM_ROOT (-1)      /* l(c_e.start - in.start | in_ep, e)   when ep e has no in-edges  */
#define TW_TERM_LAST (-2)      /* l(in.end - c_e.end | e, in_ep)       for the ep whose span ends last */

/*
 * A batch of problems, SoA.  Host code builds the (small) descriptor arrays; span arrays are the
 * bulk data.  Replaces the `{ep: [Span]}` partitions + nx.DiGraph passed at executor.py:1172-1175.
 */
typedef struct tw_batch {
  int32_t n_problems;            /* P                                                             */
  int32_t n_ep_total;            /* sum over problems of E                                        */
  int32_t n_term_total;          /* sum over problems of score terms                              */
  int32_t reserved0;
  int64_t n_in_total;
  int64_t n_out_total;
  const int64_t* prob_in_off;    /* [P+1]  in-span offset of problem p                            */
  const int32_t* prob_ep_off;    /* [P+1]  first global ep index of problem p (E = difference)    */
  const int64_t* prob_tuple_off; /* [P+1]  cumulative n_in*E: base of per-(ep,in-span) outputs    */
  const int64_t* ep_out_off;     /* [n_ep_total+1] out-span offset of (problem, ep)               */
  const int32_t* ep_term_off;    /* [n_ep_total+1] first global term index of (problem, ep).
                                    Terms of ep e, in the reference's summation order
                                    (traceweaver_v1.py:316-357): one per PRIMARY in-edge b->e in
                                    in_edges order, else one ROOT term if e has no in-edges; then
                                    always the LAST term.                                          */
  const uint32_t* ep_pred_mask;  /* [n_ep_total] bit b set: DAG edge (topo position b) -> e; every
                                    edge, primary or not, is a feasibility constraint
                                    (traceweaver_v3.py:335-347)                                    */
  const int8_t* term_src;        /* [n_term_total] b >= 0: edge term from topo position b;
                                    TW_TERM_ROOT / TW_TERM_LAST                                    */
  const int64_t* in_start;       /* [n_in_total]                                                  */
  const int64_t* in_end;         /* [n_in_total]  start_mus + duration_mus                        */
  const int64_t* out_start;      /* [n_out_total]                                                 */
  const int64_t* out_end;        /* [n_out_total]                                                 */
} tw_batch;

/* Delay-distribution parameters for one pass (replaces self.services_times, traceweaver_v1.py:118). */
#define TW_PARAMS_GAUSS_BATCHED 0 /* pass 0: one (mu, sigma) per term per 100-in-span batch (v3:1173-1178) */
#define TW_PARAMS_MIXTURE 1       /* pass 1: one GMM (or degenerate Gaussian) per term (v3:1221-1222)      */
typedef struct tw_params {
  int32_t mode;
  int32_t reserved0;
  const int64_t* prob_gauss_off; /* [P+1] record offset of problem p's [n_batches][n_terms] table   */
  const double* gauss;           /* TW_GAUSS_REC doubles per record                                 */
  const double* mix;             /* [n_term_total][TW_MIX_REC]; k = 0 means Gaussian in pc[0..2]    */
} tw_params;

/* Per-pass results (replaces the 6-tuple of traceweaver_v3.py:1229 before id translation). */
typedef struct tw_pass_out {
  int32_t* assign;        /* [prob_tuple_off[P]]  assign[tuple_off[p] + e*n_in_p + i] = index into ep
                             e's out list, -1 = ("NA","NA")                  (v1:433-455)         */
  int8_t* mis_rank;       /* [n_in_total] rank of the chosen candidate in top_k, -1 = none        */
  int32_t* n_cand;        /* [n_in_total] feasible tuples seen by the with-deletion search
                             (per_span_candidates, v3:174-178)                                    */
  double* topk_score;     /* [n_in_total][K]  with-deletion top-K (v3:1182); NaN padded; may be NULL */
  int32_t* topk_idx;      /* [K * prob_tuple_off[P]]  idx[K*(tuple_off[p] + i*E) + r*E + e]; may be NULL */
  uint8_t* topk_cnt;      /* [n_in_total] valid ranks; may be NULL                               */
  int32_t* counters;      /* [P][4]: not_best_count, cnt_unassigned, mwis_nodes_max, status       */
} tw_pass_out;

/* No-deletion scoring results (top_k_2, v3:1185 -> all_topk_assignments) and window cuts. */
typedef struct tw_score_out {
  double* topk_score;     /* [n_in_total][K] descending, NaN padded; NULL = windows only          */
  int32_t* topk_idx;      /* same layout as tw_pass_out.topk_idx                                   */
  uint8_t* topk_cnt;      /* [n_in_total]                                                         */
  int32_t* n_feasible;    /* [n_in_total] number of feasible tuples on the undeleted lists         */
  uint8_t* cut;           /* [n_in_total] 1 iff PerfectCut(i) (v3:1024-1039); cut[first]=0         */
  /* Optional (all three or none): the set of out spans that appear in SOME feasible tuple of the
   * in-span (candidates_array, v3:1043-1051), as a 64-bit map per (in-span, ep) anchored at
   * used_lo.  tw_stitch uses it to prove that no candidate of an in-span has been taken, in which
   * case the top-K on the undeleted lists IS the with-deletion top-K (v3:1182 == v3:1185).       */
  int32_t* used_lo;       /* [prob_tuple_off[P]]   used_lo[tuple_off[p] + i*E + e]                 */
  uint32_t* used_bits;    /* [2 * prob_tuple_off[P]]  two words per (in-span, ep)                  */
  uint8_t* used_wide;     /* [n_in_total] 1 = the in-span's candidates exceed 64 per ep (no map)   */
  uint32_t flags;         /* TW_SCORE_* bits                                                       */
  uint32_t reserved0;
} tw_score_out;

/* tw_score_out.flags.  The windows (cut, n_feasible, used maps) depend on the span arrays only
 * (V3:1115 builds them once, before any deletion, and both iterations reuse them).  A second
 * tw_score_topk on the same bound batch — the final top-K with the refitted parameters — may set
 * TW_SCORE_KEEP_WINDOWS: cut and used_* are then neither read nor written (the arrays the first
 * call filled stay valid), only topk_* and n_feasible are produced.                              */
#define TW_SCORE_KEEP_WINDOWS 1u

typedef struct tw_engine tw_engine;   /* opaque: bound batch, device scratch, error string       */

/* Library / device probing. */
int tw_abi_version(void);
const char* tw_last_error(void);
int tw_device_count(void);

/* Engine lifetime.  `device` is a CUDA ordinal. */
int tw_engine_create(int device, tw_engine** out);
int tw_engine_destroy(tw_engine* eng);

/* Host-side validation of descriptor arrays given as HOST pointers (span arrays ignored).
 * Mirrors the asserts at v3:1088,1198 and the engine limits. */
int tw_batch_validate_host(const tw_batch* host_desc);

/*
 * Bind a batch.  `dev` holds DEVICE pointers (all fields); `host_desc` holds HOST copies of the
 * descriptor arrays (prob_*, ep_*, term_src; its span pointers are ignored).  Validates the
 * descriptors (the asserts of v3:1088,1198 plus engine limits), rejects skip budgets
 * (n_out != n_in -> TW_ERR_UNSUPPORTED), builds the tile lists and (re)uses grow-only device scratch.
 * The arrays behind `dev` must stay alive and unchanged while bound.
 */
int tw_engine_bind(tw_engine* eng, const tw_batch* dev, const tw_batch* host_desc, void* stream);

/*
 * Bind a batch whose span times are float64 microseconds (DEVICE arrays, same layout as the tw_batch
 * span arrays; the span pointers of `dev` are ignored).  This is what executor.py --compress_factor > 1
 * produces: transforms.repeat_change_spans divides start times by the factor.  Descriptors are validated
 * as by tw_engine_bind.  Each problem p gets the smallest shift s_p >= 0 such that x * 2^s_p is an
 * integer for all its start and end times; the engine keeps X = x * 2^s_p in its own int64 buffers.
 * The conversion is exact and monotone, so windows, cuts, candidate sets and assignments are those of
 * the float64 times, and every difference the path forms equals the IEEE double difference of the two
 * times whenever that difference is exact (always inside one binade: Sterbenz).
 * After this bind the usual sequence (tw_prepare, tw_params_pass0, tw_score_topk, tw_stitch,
 * tw_delays, tw_gmm_stream_draws, tw_gmm_refit) works unchanged; every parameter, delay and mixture
 * it takes or returns is in real microseconds.  Pass-0 batch sums are formed exactly and rounded once.
 * Returns TW_ERR_INVALID for a NaN or infinite time and TW_ERR_RANGE_LIMIT when max|x| * 2^s_p >= 2^55
 * (headroom for the int64 differences and 100-element sums); tw_last_error() names the problem.
 * A later tw_engine_bind returns the engine to int64 times.  Blocks until `stream` is idle.
 */
typedef struct tw_times_f64 {
  const double* in_start;        /* [n_in_total]                                                  */
  const double* in_end;          /* [n_in_total]                                                  */
  const double* out_start;       /* [n_out_total]                                                 */
  const double* out_end;         /* [n_out_total]                                                 */
} tw_times_f64;
int tw_engine_bind_f64(tw_engine* eng, const tw_batch* dev, const tw_batch* host_desc, const tw_times_f64* dev_times,
                       void* stream);

/*
 * Batch-constant pre-kernels of the path, once per bound batch before the first pass: the
 * prev-index scan PerfectCut walks (v3:1026-1032) and the sorted end-time arrays the pass-0
 * order statistics read (v3:624-645; start times arrive sorted, end times do not).
 */
int tw_prepare(tw_engine* eng, void* stream);

/* Blocks until `stream` is idle and returns the sticky device-side status of the kernels
 * launched since the last call (TW_OK, TW_ERR_MWIS_LIMIT, TW_ERR_RANGE_LIMIT, ...). */
int tw_engine_status(tw_engine* eng, void* stream);

/* Scoring tiles of the bound batch (128 in-spans each) and how many of them the last tw_score_topk
 * handed to the sequential kernel (candidate ranges wider than the maps, score ties, NaN scores).
 * Blocks until `stream` is idle.  Either pointer may be NULL. */
int tw_engine_tile_stats(tw_engine* eng, int64_t* n_tiles, int64_t* n_redone, void* stream);

/* Number of kernels this engine has launched since creation (bench.py's gpu_launches). */
int64_t tw_engine_launch_count(const tw_engine* eng);

/*
 * Pass-0 parameters on the device: order-statistics mean/std per term per 100-in-span batch.
 * Replaces ComputeEpPairDistParams3 (traceweaver_v3.py:580-646) incl. scipy.stats.tstd.
 * gauss_out: [prob_gauss_off[P]] records of TW_GAUSS_REC doubles; prob_gauss_off (device, [P+1])
 * = cumulative n_batches_p * n_terms_p.
 */
int tw_params_pass0(tw_engine* eng, const int64_t* prob_gauss_off, double* gauss_out, void* stream);

/*
 * Candidate enumeration + scoring + top-K on the UNDELETED lists, plus perfect-cut flags.
 * Replaces FindTopKAssignments(K=5, out_span_partitions) (v3:1185, :180-465 with DfsTraverseX
 * :292-351 and ScoreAssignmentAsPerInvocationGraph v1:259-361 / GetEpPairCost v1:117-139) and
 * the pre-processing half of CreateWindows2 (v3:1041-1051 + PerfectCut :1024-1039).
 * `params` may be NULL: windows only (no scoring, topk_* untouched).
 */
int tw_score_topk(tw_engine* eng, const tw_params* params, const tw_score_out* out, void* stream);

/*
 * The sequential part of one pass: windows from cut flags (v3:1056-1076), per in-span top-K on
 * the not-yet-taken out spans (v3:1182), exact MWIS per window (BuildMISInstance v3:1252-1274 +
 * gurobi_optimods.mwis at v3:1411), assignment + deletion (AddAssignment v1:433-463).
 * `undeleted` (may be NULL) = output of tw_score_topk run with the SAME params including the used
 * maps: for every in-span none of whose candidates has been taken by an earlier window the kernel
 * adopts that top-K list instead of searching again; the result is identical either way.
 */
int tw_stitch(tw_engine* eng, const tw_params* params, const uint8_t* cut, const tw_score_out* undeleted,
              const tw_pass_out* out, void* stream);

/*
 * Score a GIVEN assignment of the bound batch (int64 or tw_engine_bind_f64 binds) under `params`
 * (either mode; pass 0 uses the record of the in-span's 100-span batch).  `assign` has the layout of
 * tw_pass_out.assign, so an engine result, a ground truth (tw_ground_truth) or any other predictor's
 * answer can be passed unchanged.  Per in-span i:
 *   code_out[i]   TW_ASSESS_* below: the lowest code whose condition holds
 *   score_out[i]  ScoreAssignmentAsPerInvocationGraph (V1:259-361) of the tuple, the same value
 *                 tw_score_topk / tw_stitch give that tuple; NaN unless code_out[i] == TW_ASSESS_SCORED
 *   margin_out[i] against `final_topk` (the no-deletion top-K of tw_score_topk under the same params):
 *                 the tuple is rank 0 -> s0 - s1 (+inf with a single candidate); else score - s0 (<= 0).
 *                 NaN when the tuple is not scored or the list is empty.  final_topk and margin_out
 *                 are both NULL or both set; only topk_score / topk_idx / topk_cnt are read.
 * Per service p: prob_sum_out[p] = sum of its scored in-spans' scores (a fixed summation order: bit
 * reproducible), prob_count_out[p * TW_ASSESS_NCODES + c] = its in-spans with code c.
 * For a float64 bind the records are rescaled as for tw_score_topk, so scores are in real units.
 */
#define TW_ASSESS_SCORED 0     /* feasible: scored                                                 */
#define TW_ASSESS_NA 1         /* -1 (("NA", "NA")) at some callee                                 */
#define TW_ASSESS_RANGE 2      /* an index outside [0, n_out) of its callee's list                 */
#define TW_ASSESS_CONTAIN 3    /* a chosen span not inside the in-span (V3:328-333)                */
#define TW_ASSESS_ORDER 4      /* c_b.end > c_e.start for a DAG edge b -> e (V3:335-347)            */
#define TW_ASSESS_NCODES 5
int tw_score_assignments(tw_engine* eng, const tw_params* params, const int32_t* assign,
                         const tw_score_out* final_topk, double* score_out, uint8_t* code_out, double* margin_out,
                         double* prob_sum_out, int32_t* prob_count_out, void* stream);

/*
 * The same for a cache-mode batch (skip budgets): tw_skip_score_assignments, declared with tw_skip_solve
 * below, takes the batch and descriptor tw_skip_solve takes and does not touch a bound batch.  `assign`
 * has the layout of tw_pass_out.assign in SORTED-list indices (the indices tw_skip_solve returns):
 * -1 = ("NA", "NA"), <= -2 = a skip span (which one does not matter: the score does not depend on it).
 *   code_out[i]   TW_ASSESS_SCORED .. TW_ASSESS_ORDER as above (containment and the DAG order are checked
 *                 between real spans, as the skip search checks them), else TW_SKIP_ASSESS_UNDEFINED
 *   score_out[i]  the skip regime's score of the tuple (V1:305-361 with skip spans): the value
 *                 tw_skip_solve lists for that tuple.  Where some budget is positive it is a MEAN OF
 *                 DENSITIES (V1:133-136), not a log-likelihood: not comparable with tw_score_assignments.
 *   margin_out[i] as above, against the in-span's top2 list (top2_score / top2_idx / top2_cnt of a
 *                 tw_skip_out; the rest of it is not read); two skip spans at one position are equal.
 * prob_sum_out[p] and prob_count_out[p * TW_SKIP_ASSESS_NCODES + c] as above.
 */
#define TW_SKIP_ASSESS_UNDEFINED 5 /* the reference raises on the tuple: all skips, a chain of skipped
                                      ancestors, or a missing services_times key (V1:264-292, :117-139) */
#define TW_SKIP_ASSESS_NCODES 6

/*
 * Delay samples implied by a pass's assignments, per term (ComputeEpPairDistParams5's
 * `durations`, traceweaver_v3.py:721-760).  delays[term_sample_off[t] + j]; NA rows are dropped
 * and counts[t] receives the number of samples.  Sample capacity of term t of problem p = n_in_p.
 */
int tw_delays(tw_engine* eng, const int32_t* assign, const int64_t* term_sample_off, double* delays,
              int32_t* counts, void* stream);

/*
 * Pass-boundary refit on the device: per term, 1-D Gaussian mixtures with 1..min(5,#unique)
 * components, BIC model selection ('diag'), final 'full' fit — the algorithm of
 * sklearn.mixture.GaussianMixture as called at traceweaver_v3.py:768-786 (k-means++ / Lloyd
 * initialisation, EM with tol 1e-3, reg_covar 1e-6, max_iter 100).  Writes n_term_total records
 * of TW_MIX_REC doubles.  Randomness: the model-selection fits consume NumPy's GLOBAL legacy
 * RandomState in the reference (never seeded by it, v3:774); here that stream is
 * RandomState(seed_select), each service starts prob_base_skip[p] random_sample() calls into it
 * (device uint32[P] or NULL = 0) and visits its terms in the order term_order (device
 * int32[n_term_total]: global term index visited q-th, grouped by problem; NULL = term order).
 * The final fit uses RandomState(100) (v3:784).  n_selected_out (device int32[n_term_total]) may
 * be NULL.
 */
int tw_gmm_refit(tw_engine* eng, const int64_t* term_sample_off, const double* delays,
                 const int32_t* counts, uint32_t seed_select, const uint32_t* prob_base_skip,
                 const int32_t* term_order, double* mix_out, int32_t* n_selected_out, void* stream);

/*
 * random_sample() calls the model-selection fits of each service would consume for the given
 * delay samples: sum over its terms of draws(min(#unique, 5)).  The reference fits GMMs on the
 * TRUE assignments first (v3:796-818, i = 0) and discards them; they only advance the stream, so
 * a drop-in caller feeds the truth delays here and passes the result as prob_base_skip above.
 */
int tw_gmm_stream_draws(tw_engine* eng, const int64_t* term_sample_off, const double* delays,
                        const int32_t* counts, uint32_t* prob_draws_out, void* stream);


/* Measurement aids of the refit's FP64 roofline (bench.py: roofline_refit).
 * tw_gmm_work: sample-component evaluations the EM sweeps of tw_gmm_refit have performed since the last
 * reset (one E+M sweep of a K-component fit over n samples counts n*K); blocks until the device is idle.
 * tw_measure_fp64_peak: dense FP64 FMA issue rate of the device in TFLOP/s (8 independent DFMA chains
 * per thread, timed with CUDA events) — the builder-measured peak the refit is quoted against. */
int tw_gmm_work(tw_engine* eng, uint64_t* em_evals_out, int reset);
int tw_measure_fp64_peak(tw_engine* eng, double* tflops_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Skip / cache mode (SURVEY.md §8 rows a11, a12, f-4).  A service some of whose outgoing lists do not
 * hold one span per incoming span (overall_skip_budget != 0, traceweaver_v3.py:1138-1158 — cache hits,
 * exps/exp2) takes ONE iteration with skip spans: TallySkipSpans (v3:853-989), BuildDistributions
 * (v3:108-172), FetchSkipFromWindow (v3:820-842), the skip branch of DfsTraverseX (v3:316-324) and
 * skip-aware, normalised scoring (traceweaver_v1.py:133-136, :264-292).
 *
 * The batch is a tw_batch whose out lists are sorted by start (stable) as TallySkipSpans leaves them
 * (v3:968-971); n_out may differ from n_in.  Because the reference builds its windows and its
 * with-deletion search on the lists in the CALLER's order (which executor.py's cache transform leaves
 * partly unsorted), that order travels as a permutation.  Result indices refer to the sorted lists;
 * a skip span is the code -2 - g, g = its index among the ep's skip spans (time windows in start
 * order, then position inside the window); tw_pass_out.assign holds -2 for ("Skip", "Skip").
 * ---------------------------------------------------------------------------------------------- */
typedef struct tw_skip_desc {
  const int64_t* prob_win_off;    /* [P+1] time windows of problem p (self.time_windows, v3:973-985,
                                     including the ones earlier services left in the instance)      */
  const int64_t* win_start;       /* [prob_win_off[P]] window starts, sorted per problem (v3:830)    */
  const int64_t* prob_cnt_off;    /* [P+1] offset into skip_count: E_p * n_win_p entries per problem */
  const int32_t* skip_count;      /* skip_count[prob_cnt_off[p] + e*n_win_p + w]: skip spans WaterFill
                                     gives ep e in window w (v3:863-917; host mirror, np.argsort ties) */
  const int64_t* prob_pair_off;   /* [P+1] offset into pair_gauss in records: (E_p+1)^2 per problem  */
  const double* pair_gauss;       /* [.][2] (mean, std) of services_times[(a, b)] after BuildDistributions,
                                     a, b: 0 = incoming endpoint, 1 + e = out ep e; NaN mean = no key */
  const uint8_t* prob_normalized; /* [P] 1 iff some budget > 0 (scores are means of densities, v3:222-227) */
  const int8_t* ep_pred_order;    /* [n_ep_total][TW_MAX_E] predecessors of the ep in in_edges order, -1 padded */
  const int32_t* out_entry_pos;   /* [n_out_total] position of sorted span j in the caller's list (ep-local) */
  const int32_t* out_sorted_of_entry; /* [n_out_total] inverse permutation                            */
} tw_skip_desc;

typedef struct tw_skip_out {
  tw_pass_out pass;       /* assign (-2 = Skip), mis_rank, n_cand, with-deletion top-K (may be NULL), counters */
  double* top2_score;     /* [n_in_total][K] top_k_2 on the undeleted lists (v3:1185), NaN padded    */
  int32_t* top2_idx;      /* layout of tw_pass_out.topk_idx                                          */
  uint8_t* top2_cnt;      /* [n_in_total]                                                            */
  uint8_t* cut;           /* [n_in_total] PerfectCut flags as the reference computes them (v3:1024-1039) */
} tw_skip_out;

/* One iteration of every problem of `dev` (DEVICE pointers; `host_desc`: HOST copies of the descriptor
 * arrays as for tw_engine_bind).  Does not touch a batch bound with tw_engine_bind. */
int tw_skip_solve(tw_engine* eng, const tw_batch* dev, const tw_batch* host_desc, const tw_skip_desc* dev_skip,
                  const tw_skip_out* out, void* stream);

/* Score a GIVEN assignment of every problem of `dev` under the model of `dev_skip` (see beside
 * tw_score_assignments).  top2 and margin_out are both NULL or both set.  Blocks until `stream` is idle. */
int tw_skip_score_assignments(tw_engine* eng, const tw_batch* dev, const tw_batch* host_desc,
                              const tw_skip_desc* dev_skip, const int32_t* assign, const tw_skip_out* top2,
                              double* score_out, uint8_t* code_out, double* margin_out, double* prob_sum_out,
                              int32_t* prob_count_out, void* stream);

/* The parent search of BuildDistributions (v3:120-168) over one service's spans merged by start
 * (stable: incoming spans first, then the out eps in topological order).  label[i]: 0 = incoming
 * (server) span, 1 + e = span of out ep e.  key_out[i] = parent_label * (E + 1) + label or -1,
 * val_out[i] = the delay sample.  All pointers DEVICE. */
int tw_build_dist_samples(tw_engine* eng, int32_t n, const int64_t* start, const int64_t* end, const int8_t* label,
                          int32_t E, int64_t large_delay, int32_t* key_out, int64_t* val_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Ground truth, invocation order and accuracy on the device (SURVEY.md §8 row f-2).  All three are
 * joins on the trace id; the loader numbers the traces densely.  These entry points read only the
 * offset tables and the out_start / out_end arrays of `dev` / `host_desc` (ep_term_off, ep_pred_mask,
 * term_src may be NULL: the callee order is not known yet when the truth is derived).
 * ---------------------------------------------------------------------------------------------- */
typedef struct tw_trace_keys {
  const int32_t* in_trace;      /* [n_in_total]  trace number of every incoming span (device)            */
  const int32_t* out_trace;     /* [n_out_total] trace number of every outgoing span (device)            */
  const int32_t* prob_trace_lo; /* [P] smallest trace number among problem p's incoming spans (device)   */
  const int32_t* prob_trace_n;  /* [P] 1 + largest - smallest (device)                                   */
  int32_t n_traces;             /* every trace number is < n_traces                                      */
  int32_t reserved0;
} tw_trace_keys;

/* utils.GetGroundTruth (helpers/utils.py:22-32): truth_out[tuple_off[p] + e*n_p + i] = position of the FIRST
 * span of callee e's list that carries in-span i's trace id, -1 if none.  host_trace_n: HOST copy of
 * prob_trace_n (sizes the join tables). */
int tw_ground_truth(tw_engine* eng, const tw_batch* dev, const tw_batch* host_desc, const tw_trace_keys* keys,
                    const int32_t* host_trace_n, int32_t* truth_out, void* stream);

/* FindOrder (executor.py:214-285): violated_out[ep0_p + a] has bit b set iff some in-span's true child at
 * callee a ends after its true child at callee b starts, i.e. the edge a -> b of the complete digraph is
 * removed.  TW_ERR_INVALID if an in-span has no child at some callee (KeyError in the reference). */
int tw_find_order(tw_engine* eng, const tw_batch* dev, const tw_batch* host_desc, const int32_t* truth,
                  uint32_t* violated_out, void* stream);

/* helpers/utils.py:62-145 on index arrays.  per_prob_out[p] = {in-spans right at every callee, in-spans
 * with some rank of topk_idx right at every callee}; e2e_out = {traces seen, traces right, traces seen,
 * traces right within the top K}.  prob_first[p] != 0 marks the services TopKAccuracyEndToEnd visits FIRST
 * (there the last in-span of a trace decides, later services can only clear it; utils.py:118-143).
 * topk_idx / topk_cnt / in_trace / prob_first may be NULL. */
int tw_accuracy(tw_engine* eng, const tw_batch* dev, const tw_batch* host_desc, const int32_t* truth,
                const int32_t* assign, const int32_t* topk_idx, const uint8_t* topk_cnt, const int32_t* in_trace,
                int32_t n_traces, const uint8_t* prob_first, uint64_t* per_prob_out, uint64_t* e2e_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TRACEWEAVER_B200_H */
