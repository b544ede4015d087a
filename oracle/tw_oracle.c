/*
 * tw_oracle.c — CPU restatement of the reference hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library; the product (traceweaver_b200/) never does and fails loudly without its CUDA
 * extension.
 *
 * What is restated: `TraceWeaverV3.FindAssignments`, method "MaxScoreBatchSubsetWithSkips", in the
 * no-skip regime (every ep has n_out == n_in, so `iterations = 2`, `dynamism = False`,
 * `normalized = False`) — /root/reference/src/trace_reconstructor/ports/python/algorithms/
 * traceweaver_v3.py (V3) and traceweaver_v1.py (V1).  Each function cites the lines it follows.
 * The restatement is deliberately LITERAL where the CUDA engine is not: it keeps per-ep
 * "remaining" lists with deletion and runs FindCutoffs (V3:182-217, including the Python
 * negative-index wrap) on them, it emulates heapq + sort(reverse=True) for the top-K order
 * (V3:305-307,461), so that agreement between engine and oracle also validates the engine's
 * claim that cutoffs never remove a feasible tuple.
 *
 * Third-party arithmetic restated here (absent from /root/reference, pinned in requirements.txt):
 *   scipy.stats.norm.logpdf  (scipy==1.14.0)        -> gauss_logpdf()
 *   scipy.stats.tstd         (scipy==1.14.0)        -> tstd10()
 *   sklearn GaussianMixture.score (scikit-learn==1.5.1) -> mix_logpdf()  (+ scipy logsumexp)
 *   gurobi_optimods.mwis     (gurobi-optimods==1.1.0) -> exact MWIS by branch and bound
 *   sklearn GaussianMixture.fit / KMeans            -> oracle/tw_oracle_gmm.c
 *
 * Parity is PINNED: tests/test_oracle_golden.py checks this file against golden vectors minted
 * by running the reference itself in the build container (tests/golden/make_goldens.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/traceweaver_b200.h"
#include "tw_oracle.h"

#define LOG_SQRT_2PI 0.91893853320467274178032973640562 /* np.log(np.sqrt(2*np.pi)) */
#define LOG_2PI 1.8378770664093453                        /* math.log(2*math.pi)     */

/* ------------------------------------------------------------------------------------------
 * Likelihood terms — GetEpPairCost, V1:117-139
 * ---------------------------------------------------------------------------------------- */

/* scipy.stats.norm.logpdf(dt, loc=mu, scale=sigma) = -x**2/2 - log(sqrt(2pi)) - log(sigma),
 * x = (dt-mu)/sigma; the std<1e-12 -> 0.001 clamp (V1:130-131) is applied when the record is
 * built, so rec = {mu, sigma, log(sigma)}. */
static double gauss_logpdf(const double* rec, double dt) {
  double x = (dt - rec[0]) / rec[1];
  return (-(x * x) / 2.0 - LOG_SQRT_2PI) - rec[2];
}

/* GaussianMixture.score(one sample) = logsumexp_k(log N_k + log w_k), V1:125-126.
 * rec = {k, pc[5], mu*pc[5], log(pc)[5], log(w)[5]}; sklearn _estimate_log_gaussian_prob 'full':
 * y = x*pc - mu*pc; -0.5*(log(2pi) + y*y) + log(pc); scipy.special.logsumexp (1.18 layout):
 * a_max + log(m) + log1p(sum_{not max} exp(a - a_max) / m), m = number of maxima. */
static double mix_logpdf(const double* rec, double dt) {
  int k = (int)rec[0];
  if (k == 0) return gauss_logpdf(rec + 1, dt);
  double a[TW_GMM_MAX_COMP];
  double amax = -INFINITY;
  for (int c = 0; c < k; ++c) {
    double y = dt * rec[1 + c] - rec[6 + c];
    a[c] = (-0.5 * (LOG_2PI + y * y) + rec[11 + c]) + rec[16 + c];
    if (a[c] > amax) amax = a[c];
  }
  double s = 0.0, m = 0.0;
  for (int c = 0; c < k; ++c) {
    if (a[c] == amax) m += 1.0;
    else s += exp(a[c] - amax);
  }
  if (s != 0.0) s = s / m;
  return log1p(s) + log(m) + amax;
}

static double term_logpdf(const tw_params* prm, int64_t gauss_base, int n_terms_p, int term_local,
                          int64_t term_global, int batch, double dt) {
  if (prm->mode == TW_PARAMS_GAUSS_BATCHED)
    return gauss_logpdf(prm->gauss + (gauss_base + (int64_t)batch * n_terms_p + term_local) * TW_GAUSS_REC, dt);
  return mix_logpdf(prm->mix + term_global * TW_MIX_REC, dt);
}

/* ------------------------------------------------------------------------------------------
 * Problem view
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int E, n_in, n_terms;
  int64_t in_off, tuple_off;
  int32_t ep0, term0;
  const int64_t *is, *ie;          /* in start / end           */
  const int64_t *os[TW_MAX_E], *oe[TW_MAX_E];
  int n_out[TW_MAX_E];
  uint32_t pred[TW_MAX_E], succ[TW_MAX_E];
  int term_lo[TW_MAX_E], term_hi[TW_MAX_E]; /* local term range of ep e */
  const int8_t* term_src;          /* local */
} prob_t;

static int view(const tw_batch* b, int p, prob_t* v) {
  memset(v, 0, sizeof *v);
  v->ep0 = b->prob_ep_off[p];
  v->E = b->prob_ep_off[p + 1] - v->ep0;
  if (v->E < 1 || v->E > TW_MAX_E) return TW_ERR_INVALID;
  v->in_off = b->prob_in_off[p];
  v->n_in = (int)(b->prob_in_off[p + 1] - v->in_off);
  v->tuple_off = b->prob_tuple_off[p];
  v->is = b->in_start + v->in_off;
  v->ie = b->in_end + v->in_off;
  v->term0 = b->ep_term_off[v->ep0];
  v->n_terms = b->ep_term_off[v->ep0 + v->E] - v->term0;
  v->term_src = b->term_src + v->term0;
  for (int e = 0; e < v->E; ++e) {
    int64_t o = b->ep_out_off[v->ep0 + e];
    v->os[e] = b->out_start + o;
    v->oe[e] = b->out_end + o;
    v->n_out[e] = (int)(b->ep_out_off[v->ep0 + e + 1] - o);
    v->pred[e] = b->ep_pred_mask[v->ep0 + e];
    v->term_lo[e] = b->ep_term_off[v->ep0 + e] - v->term0;
    v->term_hi[e] = b->ep_term_off[v->ep0 + e + 1] - v->term0;
  }
  for (int e = 0; e < v->E; ++e)
    for (int s = 0; s < v->E; ++s)
      if (v->pred[s] >> e & 1) v->succ[e] |= 1u << s;
  return TW_OK;
}

/* ------------------------------------------------------------------------------------------
 * ScoreAssignmentAsPerInvocationGraph, V1:305-361 (no skips, normalized=False).
 * c[e] = ORIGINAL index of the out span chosen for ep e.
 * ---------------------------------------------------------------------------------------- */
static double score_tuple(const prob_t* v, const tw_params* prm, int64_t gauss_base, int i,
                          const int* c) {
  int batch = i / TW_PARAM_BATCH;
  /* last_ep: max(..., key=end) keeps the FIRST maximum in tuple order (V1:314) */
  int last = 0;
  for (int e = 1; e < v->E; ++e)
    if (v->oe[e][c[e]] > v->oe[last][c[last]]) last = e;
  double cost = 0.0;
  for (int e = 0; e < v->E; ++e) {
    for (int t = v->term_lo[e]; t < v->term_hi[e]; ++t) {
      int src = v->term_src[t];
      double dt;
      if (src >= 0) dt = (double)(v->os[e][c[e]] - v->oe[src][c[src]]);       /* V1:345 */
      else if (src == TW_TERM_ROOT) dt = (double)(v->os[e][c[e]] - v->is[i]); /* V1:349-350 */
      else {                                                                  /* V1:354-355 */
        if (e != last) continue;
        dt = (double)(v->ie[i] - v->oe[e][c[e]]);
      }
      cost += term_logpdf(prm, gauss_base, v->n_terms, t, v->term0 + t, batch, dt);
    }
  }
  return cost;
}

/* ------------------------------------------------------------------------------------------
 * Remaining lists (the working copy the reference deletes from, V1:457-463)
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int* idx[TW_MAX_E]; /* original indices, ascending */
  int m[TW_MAX_E];
} rem_t;

static int rem_init(rem_t* r, const prob_t* v) {
  for (int e = 0; e < v->E; ++e) {
    r->idx[e] = (int*)malloc(sizeof(int) * (size_t)(v->n_out[e] > 0 ? v->n_out[e] : 1));
    if (!r->idx[e]) return TW_ERR_INVALID;
    for (int j = 0; j < v->n_out[e]; ++j) r->idx[e][j] = j;
    r->m[e] = v->n_out[e];
  }
  return TW_OK;
}
static void rem_free(rem_t* r, int E) {
  for (int e = 0; e < E; ++e) free(r->idx[e]);
}
static void rem_remove(rem_t* r, int e, int orig) { /* list.remove(span), V1:463 */
  int lo = 0, hi = r->m[e];
  while (lo < hi) {
    int mid = (lo + hi) / 2;
    if (r->idx[e][mid] < orig) lo = mid + 1; else hi = mid;
  }
  memmove(r->idx[e] + lo, r->idx[e] + lo + 1, sizeof(int) * (size_t)(r->m[e] - lo - 1));
  r->m[e]--;
}

/* FindCutoffs, V3:182-217, on the remaining lists.  Returns TW_ERR_INVALID where the reference
 * would raise IndexError (a successor list that is empty). */
static int find_cutoffs(const prob_t* v, const rem_t* r, int i, int* lo, int* hi) {
  for (int e = v->E - 1; e >= 0; --e) { /* reverse topological order */
    int64_t exit_t = v->ie[i];
    for (int s = 0; s < v->E; ++s) {
      if (!(v->succ[e] >> s & 1)) continue;
      int h = hi[s];
      if (h < 0) h += r->m[s]; /* Python negative index: [-1] is the last element */
      if (h < 0 || h >= r->m[s]) return TW_ERR_INVALID;
      int64_t st = v->os[s][r->idx[s][h]];
      if (st < exit_t) exit_t = st;
    }
    int a = 0, bnd = r->m[e];
    while (a < bnd) { /* bisect_left(starts, in.start) */
      int mid = (a + bnd) / 2;
      if (v->os[e][r->idx[e][mid]] < v->is[i]) a = mid + 1; else bnd = mid;
    }
    lo[e] = a;
    a = 0; bnd = r->m[e];
    while (a < bnd) { /* bisect_right(starts, exit) */
      int mid = (a + bnd) / 2;
      if (exit_t < v->os[e][r->idx[e][mid]]) bnd = mid; else a = mid + 1;
    }
    hi[e] = a - 1;
  }
  return TW_OK;
}

/* ------------------------------------------------------------------------------------------
 * heapq emulation for (score, stack) pairs — V3:305-307 (push, pop when len > K), V3:461
 * (sort(reverse=True)).  `lt` reproduces tuple/list comparison: score first; on equal scores the
 * first position whose span object differs decides by Span.__lt__ = start_mus (spans.py:51).
 * ---------------------------------------------------------------------------------------- */
typedef struct { double score; int c[TW_MAX_E]; } cand_t;

static int cand_lt(const prob_t* v, const cand_t* a, const cand_t* b) {
  if (a->score < b->score) return 1;
  if (a->score > b->score) return 0;
  if (a->score != b->score) return 0; /* NaN */
  for (int e = 0; e < v->E; ++e)
    if (a->c[e] != b->c[e]) return v->os[e][a->c[e]] < v->os[e][b->c[e]];
  return 0;
}
static void sift_down(const prob_t* v, cand_t* h, int startpos, int pos) {
  cand_t item = h[pos];
  while (pos > startpos) {
    int parent = (pos - 1) >> 1;
    if (cand_lt(v, &item, &h[parent])) { h[pos] = h[parent]; pos = parent; continue; }
    break;
  }
  h[pos] = item;
}
static void sift_up(const prob_t* v, cand_t* h, int n, int pos) {
  int endpos = n, startpos = pos;
  cand_t item = h[pos];
  int child = 2 * pos + 1;
  while (child < endpos) {
    int right = child + 1;
    if (right < endpos && !cand_lt(v, &h[child], &h[right])) child = right;
    h[pos] = h[child];
    pos = child;
    child = 2 * pos + 1;
  }
  h[pos] = item;
  sift_down(v, h, startpos, pos);
}
typedef struct { cand_t h[TW_K + 1]; int n; } heap_t;
static void heap_offer(const prob_t* v, heap_t* hp, const cand_t* c) {
  hp->h[hp->n++] = *c;
  sift_down(v, hp->h, 0, hp->n - 1);
  if (hp->n > TW_K) { /* heappop */
    cand_t last = hp->h[--hp->n];
    if (hp->n > 0) { hp->h[0] = last; sift_up(v, hp->h, hp->n, 0); }
  }
}
/* list.sort(reverse=True): stable w.r.t. the reversed relation — equal elements keep their
 * original relative order.  Insertion sort, descending, stable. */
static void heap_sorted_desc(const prob_t* v, heap_t* hp) {
  for (int a = 1; a < hp->n; ++a) {
    cand_t x = hp->h[a];
    int j = a - 1;
    while (j >= 0 && cand_lt(v, &hp->h[j], &x)) { hp->h[j + 1] = hp->h[j]; --j; }
    hp->h[j + 1] = x;
  }
}

/* ------------------------------------------------------------------------------------------
 * DfsTraverseX (V3:292-351) / DfsTraverse3 (V3:236-288) on remaining lists.
 * mark != NULL: record every out span that appears in a feasible tuple (candidates_array,
 * V3:1043-1051).  prm == NULL: unscored enumeration.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  const prob_t* v; const rem_t* r; const tw_params* prm; int64_t gauss_base;
  int i; const int *lo, *hi; int c[TW_MAX_E];
  heap_t* heap; int64_t leaves; uint8_t** mark;
} dfs_t;

static void dfs(dfs_t* d, int e) {
  const prob_t* v = d->v;
  if (e == v->E) {
    d->leaves++;
    if (d->mark) for (int q = 0; q < v->E; ++q) d->mark[q][d->c[q]] = 1;
    if (d->prm) {
      cand_t cd;
      cd.score = score_tuple(v, d->prm, d->gauss_base, d->i, d->c);
      memcpy(cd.c, d->c, sizeof cd.c);
      heap_offer(v, d->heap, &cd);
    }
    return;
  }
  for (int x = d->lo[e]; x <= d->hi[e] && x < d->r->m[e]; ++x) {
    if (x < 0) continue;
    int o = d->r->idx[e][x];
    if (v->is[d->i] > v->os[e][o] || v->oe[e][o] > v->ie[d->i]) continue; /* V3:328-333 */
    int ok = 1;
    for (int bq = 0; bq < e; ++bq)                                           /* V3:335-347 */
      if ((v->pred[e] >> bq & 1) && v->oe[bq][d->c[bq]] > v->os[e][o]) { ok = 0; break; }
    if (!ok) continue;
    d->c[e] = o;
    dfs(d, e + 1);
  }
}

/* ------------------------------------------------------------------------------------------
 * Windows: CreateWindows2, V3:1020-1078.
 * cut[i] = PerfectCut(i) for 1 <= i <= n-2 (0 elsewhere); win_end[i] = 1 iff a window ends at i.
 * n_feasible[i] = number of feasible tuples on the undeleted lists.
 * ---------------------------------------------------------------------------------------- */
static void windows_from_cuts(int n, const uint8_t* cut, uint8_t* win_end) {
  memset(win_end, 0, (size_t)n);
  int current_count = 1;
  for (int i = 0; i < n; ++i) {
    if (i != 0) {
      if (i == n - 1) { current_count = 0; win_end[i] = 1; }
      else if (cut[i]) { current_count = 0; win_end[i - 1] = 1; }
      else if (current_count == TW_MAX_WINDOW) { current_count = 0; win_end[i] = 1; }
    }
    current_count += 1;
  }
  if (n == 1) win_end[0] = 0; /* the reference creates no window for a single in-span */
}

int two_score_problem(const tw_batch* b, int p, const tw_params* prm, const tw_score_out* out) {
  prob_t v; int rc = view(b, p, &v);
  if (rc) return rc;
  rem_t r; if ((rc = rem_init(&r, &v))) return rc;
  int n = v.n_in;
  int64_t gauss_base = prm && prm->mode == TW_PARAMS_GAUSS_BATCHED ? prm->prob_gauss_off[p] : 0;
  /* per in-span marks: bitmap over all out spans is too big to keep for every i; the cut only
     ever compares i with prev_index, so keep marks of "prev" and "current". */
  uint8_t *mk_prev[TW_MAX_E], *mk_cur[TW_MAX_E], *mk_tmp[TW_MAX_E];
  for (int e = 0; e < v.E; ++e) {
    mk_prev[e] = (uint8_t*)calloc((size_t)v.n_out[e] + 1, 1);
    mk_cur[e] = (uint8_t*)calloc((size_t)v.n_out[e] + 1, 1);
    mk_tmp[e] = (uint8_t*)calloc((size_t)v.n_out[e] + 1, 1);
  }
  int prev_index = 0;
  int lo[TW_MAX_E], hi[TW_MAX_E];
  for (int i = 0; i < n; ++i) {
    rc = find_cutoffs(&v, &r, i, lo, hi);
    if (rc) break;
    heap_t heap; heap.n = 0;
    for (int e = 0; e < v.E; ++e) memset(mk_cur[e], 0, (size_t)v.n_out[e]);
    dfs_t d = {&v, &r, prm, gauss_base, i, lo, hi, {0}, &heap, 0, mk_cur};
    dfs(&d, 0);
    out->n_feasible[v.in_off + i] = (int32_t)d.leaves;
    if (prm && out->topk_score) {
      heap_sorted_desc(&v, &heap);
      out->topk_cnt[v.in_off + i] = (uint8_t)heap.n;
      for (int k = 0; k < TW_K; ++k) {
        out->topk_score[(v.in_off + i) * TW_K + k] = k < heap.n ? heap.h[k].score : NAN;
        for (int e = 0; e < v.E; ++e)
          out->topk_idx[TW_K * (v.tuple_off + (int64_t)i * v.E) + k * v.E + e] = k < heap.n ? heap.h[k].c[e] : -1;
      }
    }
    /* PerfectCut(i), V3:1024-1039.  prev_index is the latest-ending in-span among [0, i-1],
       ties to the later one; it is only advanced inside PerfectCut, which is called for
       1 <= i <= n-2. */
    uint8_t cutflag = 0;
    if (i >= 1 && i <= n - 2) {
      if (i == 1) prev_index = 0;
      else if (v.ie[i - 1] >= v.ie[prev_index]) prev_index = i - 1;
      /* marks of prev_index: recompute (cheap; keeps memory O(n_out)) */
      int lo2[TW_MAX_E], hi2[TW_MAX_E];
      rc = find_cutoffs(&v, &r, prev_index, lo2, hi2);
      if (rc) break;
      for (int e = 0; e < v.E; ++e) memset(mk_tmp[e], 0, (size_t)v.n_out[e]);
      dfs_t d2 = {&v, &r, NULL, 0, prev_index, lo2, hi2, {0}, NULL, 0, mk_tmp};
      dfs(&d2, 0);
      int disjoint = 1;
      for (int e = 0; e < v.E && disjoint; ++e)
        for (int j = 0; j < v.n_out[e]; ++j)
          if (mk_tmp[e][j] && mk_cur[e][j]) { disjoint = 0; break; }
      cutflag = (uint8_t)(disjoint && v.ie[prev_index] <= v.ie[i]);
    }
    out->cut[v.in_off + i] = cutflag;
  }
  for (int e = 0; e < v.E; ++e) { free(mk_prev[e]); free(mk_cur[e]); free(mk_tmp[e]); }
  rem_free(&r, v.E);
  return rc;
}

/* ------------------------------------------------------------------------------------------
 * Exact MWIS — BuildMISInstance V3:1252-1274 + the solver call V3:1411.
 * Vertices (ind, rank) with weight 10000+score; edges: same ind, or a shared out span at the
 * same tuple position (AssignmentIntersect V3:1276-1281).  Branch and bound over in-spans in
 * window order: pick one compatible candidate or none.  Vertices with weight <= 0 are never
 * chosen (SURVEY A.9 item 6).  Ties (totals within TW_MWIS_TIE_TOL; Gurobi's choice is arbitrary
 * there) go to the first leaf of this depth-first order.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  const prob_t* v; int nw;
  const heap_t* cand;            /* [nw] sorted desc */
  double w[TW_WINDOW_CAP][TW_K];
  double ub_suffix[TW_WINDOW_CAP + 1];
  int cur[TW_WINDOW_CAP], best[TW_WINDOW_CAP];
  double best_w; int64_t nodes;
} mwis_t;

static int mw_conflict(const mwis_t* m, int a, int ra, int bq, int rb) {
  for (int e = 0; e < m->v->E; ++e)
    if (m->cand[a].h[ra].c[e] == m->cand[bq].h[rb].c[e]) return 1;
  return 0;
}
#define TWO_MWIS_NODE_LIMIT 20000000LL /* give up loudly instead of searching for hours */
static void mw_rec(mwis_t* m, int k, double cur_w) {
  if (m->nodes > TWO_MWIS_NODE_LIMIT) return;
  m->nodes++;
  if (k == m->nw) {
    if (cur_w > m->best_w + TW_MWIS_TIE_TOL) { m->best_w = cur_w; memcpy(m->best, m->cur, sizeof(int) * (size_t)m->nw); }
    return;
  }
  if (cur_w + m->ub_suffix[k] <= m->best_w + TW_MWIS_TIE_TOL) return;
  for (int r = 0; r < m->cand[k].n; ++r) {
    if (!(m->w[k][r] > 0.0)) continue;
    int ok = 1;
    for (int a = 0; a < k && ok; ++a)
      if (m->cur[a] >= 0 && mw_conflict(m, a, m->cur[a], k, r)) ok = 0;
    if (!ok) continue;
    m->cur[k] = r;
    mw_rec(m, k + 1, cur_w + m->w[k][r]);
  }
  m->cur[k] = -1;
  mw_rec(m, k + 1, cur_w);
}
static int64_t mwis_solve(const prob_t* v, const heap_t* cand, int nw, int* chosen) {
  mwis_t m; m.v = v; m.nw = nw; m.cand = cand; m.best_w = -1.0; m.nodes = 0;
  for (int k = 0; k < nw; ++k) { m.cur[k] = -1; m.best[k] = -1; }
  m.ub_suffix[nw] = 0.0;
  for (int k = nw - 1; k >= 0; --k) {
    double mx = 0.0;
    for (int r = 0; r < cand[k].n; ++r) {
      m.w[k][r] = TW_WEIGHT_OFFSET + cand[k].h[r].score;
      if (m.w[k][r] > mx) mx = m.w[k][r];
    }
    m.ub_suffix[k] = m.ub_suffix[k + 1] + mx;
  }
  mw_rec(&m, 0, 0.0);
  memcpy(chosen, m.best, sizeof(int) * (size_t)nw);
  return m.nodes;
}

/* ------------------------------------------------------------------------------------------
 * One pass of the hot loop, V3:1159-1219.
 * ---------------------------------------------------------------------------------------- */
int two_stitch_problem(const tw_batch* b, int p, const tw_params* prm, const uint8_t* cut,
                       const tw_pass_out* out) {
  prob_t v; int rc = view(b, p, &v);
  if (rc) return rc;
  rem_t r; if ((rc = rem_init(&r, &v))) return rc;
  int n = v.n_in;
  int64_t gauss_base = prm->mode == TW_PARAMS_GAUSS_BATCHED ? prm->prob_gauss_off[p] : 0;
  uint8_t* win_end = (uint8_t*)malloc((size_t)n);
  windows_from_cuts(n, cut + v.in_off, win_end);
  heap_t window[TW_WINDOW_CAP];
  int nw = 0, ws = 0;
  int32_t not_best = 0, unassigned = 0; int64_t max_nodes = 0;
  int lo[TW_MAX_E], hi[TW_MAX_E];
  /* in-spans never reached by a window end (only possible for n == 1) stay unassigned */
  for (int e = 0; e < v.E; ++e)
    for (int i = 0; i < n; ++i) out->assign[v.tuple_off + (int64_t)e * n + i] = -1;
  for (int i = 0; i < n; ++i) out->mis_rank[v.in_off + i] = -1;
  for (int i = 0; i < n && !rc; ++i) {
    rc = find_cutoffs(&v, &r, i, lo, hi);
    if (rc) break;
    heap_t* hp = &window[nw];
    hp->n = 0;
    dfs_t d = {&v, &r, prm, gauss_base, i, lo, hi, {0}, hp, 0, NULL};
    dfs(&d, 0);
    heap_sorted_desc(&v, hp);
    out->n_cand[v.in_off + i] = (int32_t)d.leaves;
    if (out->topk_score) {
      out->topk_cnt[v.in_off + i] = (uint8_t)hp->n;
      for (int k = 0; k < TW_K; ++k) {
        out->topk_score[(v.in_off + i) * TW_K + k] = k < hp->n ? hp->h[k].score : NAN;
        for (int e = 0; e < v.E; ++e)
          out->topk_idx[TW_K * (v.tuple_off + (int64_t)i * v.E) + k * v.E + e] = k < hp->n ? hp->h[k].c[e] : -1;
      }
    }
    nw++;
    if (win_end[i]) { /* V3:1192-1219 */
      int chosen[TW_WINDOW_CAP];
      int64_t nodes = mwis_solve(&v, window, nw, chosen);
      if (nodes > TWO_MWIS_NODE_LIMIT) { rc = TW_ERR_MWIS_LIMIT; break; }
      if (nodes > max_nodes) max_nodes = nodes;
      for (int k = 0; k < nw; ++k) {
        int ii = ws + k;
        out->mis_rank[v.in_off + ii] = (int8_t)chosen[k];
        if (chosen[k] != 0) not_best++;           /* V3:1201-1207 */
        if (chosen[k] < 0) { unassigned++; continue; }
        for (int e = 0; e < v.E; ++e) {
          int o = window[k].h[chosen[k]].c[e];
          out->assign[v.tuple_off + (int64_t)e * n + ii] = o;
          rem_remove(&r, e, o);                   /* V1:457-463 */
        }
      }
      nw = 0; ws = i + 1;
    } else if (nw >= TW_WINDOW_CAP) { rc = TW_ERR_INVALID; }
  }
  if (out->counters) {
    out->counters[p * 4 + 0] = not_best;
    out->counters[p * 4 + 1] = unassigned;
    out->counters[p * 4 + 2] = (int32_t)(max_nodes > 0x7fffffff ? 0x7fffffff : max_nodes);
    out->counters[p * 4 + 3] = rc;
  }
  free(win_end);
  rem_free(&r, v.E);
  return rc;
}

/* ------------------------------------------------------------------------------------------
 * A GIVEN assignment scored: ScoreAssignmentAsPerInvocationGraph (V1:259-361) of in-span i's
 * tuple after the feasibility checks of DfsTraverseX (V3:328-347).  code[i]: TW_ASSESS_*, the
 * lowest whose condition holds; score[i] NaN unless scored.  prob_sum / prob_count: the scored
 * in-spans' scores added in in-span order, and the in-spans per code.
 * ---------------------------------------------------------------------------------------- */
int two_assess_problem(const tw_batch* b, int p, const tw_params* prm, const int32_t* assign, double* score,
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

/* ------------------------------------------------------------------------------------------
 * Pass-0 parameters: ComputeEpPairDistParams3, V3:580-646.
 * ---------------------------------------------------------------------------------------- */
static int cmp_i64(const void* a, const void* b) {
  int64_t x = *(const int64_t*)a, y = *(const int64_t*)b;
  return x < y ? -1 : x > y;
}
/* np.sum over a contiguous float64 vector of length n <= 10: numpy's pairwise_sum (8 lanes). */
static double np_sum(const double* a, int n) {
  if (n < 8) { double r = 0.0; for (int i = 0; i < n; ++i) r += a[i]; return r; }
  double r[8]; for (int j = 0; j < 8; ++j) r[j] = a[j];
  int i = 8;
  for (; i < n - (n % 8); i += 8) for (int j = 0; j < 8; ++j) r[j] += a[i + j];
  double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) res += a[i];
  return res;
}
/* scipy.stats.tstd(batch_means): sqrt(mean((x-mean)^2) * n/(n-1)); NaN for n == 1 (A.9 item 9). */
static double tstd(const double* x, int n) {
  double mean = np_sum(x, n) / (double)n;
  double d[TW_PARAM_NBATCHES];
  for (int i = 0; i < n; ++i) { double t = x[i] - mean; d[i] = t * t; }
  double var = np_sum(d, n) / (double)n;
  if (n - 1 <= 0) return NAN;
  var *= (double)n / (double)(n - 1);
  return sqrt(var);
}
static void dist_params(const int64_t* t1, const int64_t* t2, int s, int e, double* rec) {
  int m = e - s;
  int64_t num = 0;
  for (int j = s; j < e; ++j) num += t2[j] - t1[j];
  double mean = (double)num / (double)m;              /* V3:594 (exact int / int) */
  int bs = (m + TW_PARAM_NBATCHES - 1) / TW_PARAM_NBATCHES; /* V3:600 */
  double bm[TW_PARAM_NBATCHES]; int nb = 0;
  for (int q = 0; q < TW_PARAM_NBATCHES; ++q) {
    int a = s + q * bs, z = s + (q + 1) * bs; if (z > e) z = e;
    if (z - a > 0) {
      int64_t nn = 0;
      for (int j = a; j < z; ++j) nn += t2[j] - t1[j];
      bm[nb++] = (double)nn / (double)(z - a);
    }
  }
  double std = sqrt((double)bs) * tstd(bm, nb);       /* V3:611 */
  if (std < 1.0e-12) std = 0.001;                     /* V1:130-131 (applied at use) */
  rec[0] = mean; rec[1] = std; rec[2] = log(std);
}

int two_params_pass0(const tw_batch* b, int p, const int64_t* prob_gauss_off, double* gauss) {
  prob_t v; int rc = view(b, p, &v);
  if (rc) return rc;
  int n = v.n_in;
  for (int e = 0; e < v.E; ++e) if (v.n_out[e] != n) return TW_ERR_UNSUPPORTED;
  int64_t* in_s = (int64_t*)malloc(sizeof(int64_t) * (size_t)n * 2);
  int64_t* in_e = in_s + n;
  memcpy(in_s, v.is, sizeof(int64_t) * (size_t)n); memcpy(in_e, v.ie, sizeof(int64_t) * (size_t)n);
  qsort(in_s, (size_t)n, sizeof(int64_t), cmp_i64); qsort(in_e, (size_t)n, sizeof(int64_t), cmp_i64);
  int64_t* os[TW_MAX_E]; int64_t* oe[TW_MAX_E];
  for (int e = 0; e < v.E; ++e) {
    os[e] = (int64_t*)malloc(sizeof(int64_t) * (size_t)n * 2); oe[e] = os[e] + n;
    memcpy(os[e], v.os[e], sizeof(int64_t) * (size_t)n); memcpy(oe[e], v.oe[e], sizeof(int64_t) * (size_t)n);
    qsort(os[e], (size_t)n, sizeof(int64_t), cmp_i64); qsort(oe[e], (size_t)n, sizeof(int64_t), cmp_i64);
  }
  int nb = (n + TW_PARAM_BATCH - 1) / TW_PARAM_BATCH;
  for (int bt = 0; bt < nb; ++bt) {
    int s = bt * TW_PARAM_BATCH, z = s + TW_PARAM_BATCH; if (z > n) z = n;
    for (int e = 0; e < v.E; ++e)
      for (int t = v.term_lo[e]; t < v.term_hi[e]; ++t) {
        double* rec = gauss + (prob_gauss_off[p] + (int64_t)bt * v.n_terms + t) * TW_GAUSS_REC;
        int src = v.term_src[t];
        if (src >= 0) dist_params(oe[src], os[e], s, z, rec);           /* V3:640-642 */
        else if (src == TW_TERM_ROOT) dist_params(in_s, os[e], s, z, rec); /* V3:623-626 */
        else dist_params(oe[e], in_e, s, z, rec);                        /* V3:644-646 */
      }
  }
  for (int e = 0; e < v.E; ++e) free(os[e]);
  free(in_s);
  return TW_OK;
}

/* ------------------------------------------------------------------------------------------
 * Delay samples implied by assignments: ComputeEpPairDistParams5's `durations`, V3:721-760.
 * ---------------------------------------------------------------------------------------- */
int two_delays(const tw_batch* b, int p, const int32_t* assign, const int64_t* term_sample_off,
               double* delays, int32_t* counts) {
  prob_t v; int rc = view(b, p, &v);
  if (rc) return rc;
  int n = v.n_in;
  for (int e = 0; e < v.E; ++e)
    for (int t = v.term_lo[e]; t < v.term_hi[e]; ++t) {
      int src = v.term_src[t];
      double* dst = delays + term_sample_off[v.term0 + t];
      int cnt = 0;
      for (int i = 0; i < n; ++i) {
        int ce = assign[v.tuple_off + (int64_t)e * n + i];
        if (ce < 0) continue;
        if (src >= 0) {
          int cb = assign[v.tuple_off + (int64_t)src * n + i];
          if (cb < 0) continue;
          dst[cnt++] = (double)(v.os[e][ce] - v.oe[src][cb]);   /* mapping_type 2 */
        } else if (src == TW_TERM_ROOT) dst[cnt++] = (double)(v.os[e][ce] - v.is[i]); /* type 1 */
        else dst[cnt++] = (double)(v.ie[i] - v.oe[e][ce]);       /* type 3 */
      }
      counts[v.term0 + t] = cnt;
    }
  return TW_OK;
}

int two_windows_from_cuts(int n, const uint8_t* cut, uint8_t* win_end) {
  windows_from_cuts(n, cut, win_end);
  return TW_OK;
}
