/*
 * tw_oracle_gmm.c — CPU restatement of the pass-boundary refit.  TEST INFRASTRUCTURE ONLY.
 *
 * Reference call site: ComputeEpPairDistParams5, traceweaver_v3.py:764-786
 *     max_n = min(len(np.unique(durations)), 5)
 *     for n in 1..max_n: GaussianMixture(n_components=n, covariance_type='diag').fit(durations)
 *     n_selected = argmin BIC
 *     g = GaussianMixture(n_components=n_selected, random_state=100).fit(durations)   # 'full'
 *
 * The algorithm lives in a third-party dependency that is not under /root/reference:
 * scikit-learn==1.5.1 (requirements.txt:22) — sklearn/mixture/_base.py (fit_predict: k-means
 * initialisation, EM until |delta lower bound| < tol=1e-3, max_iter=100, n_init=1),
 * sklearn/mixture/_gaussian_mixture.py (_estimate_gaussian_parameters, reg_covar=1e-6,
 * _estimate_log_gaussian_prob for 'diag' and 'full', bic), sklearn/cluster/_kmeans.py
 * (_kmeans_plusplus with n_local_trials = 2+int(ln k), _kmeans_single_lloyd with
 * tol = 1e-4*var(X), max_iter=300) and numpy's legacy RandomState (MT19937, random_sample,
 * choice(p=...)).  This file restates those published algorithms for one feature.  Randomness:
 * the model-selection fits draw from NumPy's GLOBAL RandomState (the reference never seeds it,
 * SURVEY A.9 item 7) — here an MT19937 stream seeded with `seed_select` and advanced by
 * `rng_skip` random_sample() calls; the final fit uses a fresh RandomState(100).
 *
 * Floating-point summation order of BLAS dot products inside sklearn is not reproducible, so
 * parameters agree to ~1e-9 relative, not bit for bit; tests/test_oracle_gmm.py pins this file
 * against the GaussianMixture objects recorded in the golden fixtures.
 */
#include <math.h>
#include <stdio.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/traceweaver_b200.h"
#include "tw_oracle.h"

#define LOG_2PI 1.8378770664093453
#define REG_COVAR 1e-6
#define EM_TOL 1e-3
#define EM_MAX_ITER 100
#define KM_MAX_ITER 300
#define KM_TOL 1e-4
#define DBL_EPS 2.220446049250313e-16

/* The accumulators of every sum.  The default build keeps them double; the twin build
 * (libtw_oracle_gmm_ld.so, -DTW_GMM_ACC="long double") widens them, so that a term whose discrete
 * decisions or parameters move between the two builds is known to depend on summation order. */
#ifndef TW_GMM_ACC
#define TW_GMM_ACC double
#endif
typedef TW_GMM_ACC acc_t;

/* what one fit decided (two_gmm_refit_record): a row of TW_GMM_REC_FIELDS int32 */
enum { R_STATUS, R_LLOYD_ITER, R_LLOYD_STRICT, R_RELOC, R_EM_ITER, R_EM_CONVERGED, R_REPLAY, R_LLOYD_TIES,
       TW_GMM_REC_FIELDS };
typedef int32_t fitrec_t[TW_GMM_REC_FIELDS];

/* ---- numpy legacy RandomState ----------------------------------------------------------- */
typedef struct { uint32_t mt[624]; int idx; } mt_t;

static void mt_seed(mt_t* r, uint32_t seed) { /* init_genrand */
  r->mt[0] = seed;
  for (int i = 1; i < 624; ++i) r->mt[i] = 1812433253u * (r->mt[i - 1] ^ (r->mt[i - 1] >> 30)) + (uint32_t)i;
  r->idx = 624;
}
static uint32_t mt_next(mt_t* r) {
  if (r->idx >= 624) {
    for (int k = 0; k < 624; ++k) {
      uint32_t y = (r->mt[k] & 0x80000000u) | (r->mt[(k + 1) % 624] & 0x7fffffffu);
      r->mt[k] = r->mt[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    r->idx = 0;
  }
  uint32_t y = r->mt[r->idx++];
  y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
  return y;
}
static double mt_random_sample(mt_t* r) {
  uint32_t a = mt_next(r) >> 5, b = mt_next(r) >> 6;
  return (a * 67108864.0 + b) / 9007199254740992.0;
}

/* np.sum / np.mean over a contiguous float64 vector: pairwise summation, blocks of 128, 8 lanes */
static acc_t pw_acc(const double* a, int n) {
  if (n < 8) { acc_t r = 0.0; for (int i = 0; i < n; ++i) r += a[i]; return r; }
  if (n <= 128) {
    acc_t r[8]; for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8) for (int j = 0; j < 8; ++j) r[j] += a[i + j];
    acc_t res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a[i];
    return res;
  }
  int n2 = n / 2; n2 -= n2 % 8;
  return pw_acc(a, n2) + pw_acc(a + n2, n - n2);
}
static double pw_sum(const double* a, int n) { return (double)pw_acc(a, n); }

typedef struct {
  int k;
  double w[TW_GMM_MAX_COMP], mu[TW_GMM_MAX_COMP], cov[TW_GMM_MAX_COMP], pc[TW_GMM_MAX_COMP];
  int n_iter, converged;
} gmm_t;

/* ---- k-means (labels only matter downstream) -------------------------------------------- */
/* nearest centre of x (first minimum); *tie += 1 when the runner-up's c^2 - 2 x c is within 1e-12 of the
 * terms' size: such a label follows the last bits of the centres, i.e. the summation order behind them */
static int nearest_centre(const double* centers, const double* cn, int k, double x, int32_t* tie) {
  int lab = 0; double best = cn[0] + (-2.0 * (x * centers[0])), second = INFINITY, scale = fabs(cn[0]);
  for (int j = 1; j < k; ++j) {
    double d = cn[j] + (-2.0 * (x * centers[j]));
    if (fabs(cn[j]) > scale) scale = fabs(cn[j]);
    if (d < best) { second = best; best = d; lab = j; }
    else if (d < second) second = d;
  }
  double sx = 2.0 * fabs(x) * sqrt(scale);
  if (sx > scale) scale = sx;
  if (k > 1 && second - best <= 1e-12 * scale) ++*tie;
  return lab;
}

static double sq_dist(double c, double c2, double x, double x2) { /* _euclidean_distances */
  double d = -2.0 * (c * x);
  d += c2; d += x2;
  return d > 0.0 ? d : 0.0;
}

static void kmeans_labels(const double* x_in, int n, int k, mt_t* rng, int* labels, double* work /* 4n */,
                          int32_t* fr) {
  double* x = work; double* x2 = work + n; double* closest = work + 2 * n; double* tmp = work + 3 * n;
  double mean = pw_sum(x_in, n) / (double)n;
  for (int i = 0; i < n; ++i) { x[i] = x_in[i] - mean; x2[i] = x[i] * x[i]; }
  /* tolerance: np.mean(np.var(X, axis=0)) * tol, computed before centering */
  double var;
  { double* d = tmp; double m0 = pw_sum(x_in, n) / (double)n;
    for (int i = 0; i < n; ++i) { double t = x_in[i] - m0; d[i] = t * t; }
    var = pw_sum(d, n) / (double)n; }
  double tol = var * KM_TOL;

  /* k-means++ seeding (_kmeans_plusplus) */
  double centers[TW_GMM_MAX_COMP];
  acc_t centers_new[TW_GMM_MAX_COMP], wsum[TW_GMM_MAX_COMP];
  {
    /* random_state.choice(n, p = 1/n): cdf = cumsum(p); cdf /= cdf[-1]; searchsorted(u, 'right') */
    double u = mt_random_sample(rng);
    /* the device's first_centre (tw_core.cuh) replays NumPy's sum only within this band of an integer */
    { double un = u * (double)n, bound = 1e-6, b2 = (double)n * ((double)n + 5.0) * 0x1p-52;
      if (b2 > bound) bound = b2;
      fr[R_REPLAY] = fabs(un - rint(un)) < bound; }
    double p = 1.0 / (double)n, last = 0.0;
    { double c = 0.0; for (int i = 0; i < n; ++i) c += p; last = c; }
    int id = n - 1; double c = 0.0;
    for (int i = 0; i < n; ++i) { c += p; if (c / last > u) { id = i; break; } }
    centers[0] = x[id];
    double c2 = centers[0] * centers[0];
    for (int i = 0; i < n; ++i) closest[i] = sq_dist(centers[0], c2, x[i], x2[i]);
    acc_t pot_a = 0.0; for (int i = 0; i < n; ++i) pot_a += closest[i];
    double pot = (double)pot_a;
    int trials = 2 + (int)log((double)k);
    for (int cidx = 1; cidx < k; ++cidx) {
      double rv[8]; int cand[8];
      for (int t = 0; t < trials; ++t) rv[t] = mt_random_sample(rng) * pot;
      /* np.searchsorted(np.cumsum(closest), rand_vals) (side='left'), clipped */
      for (int t = 0; t < trials; ++t) {
        acc_t cs = 0.0; int found = n - 1;
        for (int i = 0; i < n; ++i) { cs += closest[i]; if (cs >= rv[t]) { found = i; break; } }
        cand[t] = found;
      }
      int best_t = 0; double best_pot = INFINITY;
      for (int t = 0; t < trials; ++t) {
        double cc = x[cand[t]], cc2 = cc * cc;
        acc_t pt = 0.0;
        for (int i = 0; i < n; ++i) {
          double d = sq_dist(cc, cc2, x[i], x2[i]);
          pt += d < closest[i] ? d : closest[i];
        }
        if ((double)pt < best_pot) { best_pot = (double)pt; best_t = t; }
      }
      double cc = x[cand[best_t]], cc2 = cc * cc;
      for (int i = 0; i < n; ++i) {
        double d = sq_dist(cc, cc2, x[i], x2[i]);
        if (d < closest[i]) closest[i] = d;
      }
      pot = best_pot;
      centers[cidx] = cc;
    }
  }
  /* Lloyd (_kmeans_single_lloyd) */
  int* labels_old = (int*)tmp; /* n ints fit in n doubles */
  for (int i = 0; i < n; ++i) { labels[i] = -1; labels_old[i] = -1; }
  int strict = 0;
  for (int it = 0; it < KM_MAX_ITER; ++it) {
    double cn[TW_GMM_MAX_COMP];
    for (int j = 0; j < k; ++j) { cn[j] = centers[j] * centers[j]; centers_new[j] = 0.0; wsum[j] = 0.0; }
    for (int i = 0; i < n; ++i) {
      int lab = nearest_centre(centers, cn, k, x[i], &fr[R_LLOYD_TIES]);
      labels[i] = lab; centers_new[lab] += x[i]; wsum[lab] += 1.0;
    }
    /* _relocate_empty_clusters_dense: move the farthest points into empty clusters */
    for (int j = 0; j < k; ++j) {
      if (wsum[j] != 0.0) continue;
      int far = 0; double fd = -1.0;
      for (int i = 0; i < n; ++i) { double d = (x[i] - centers[labels[i]]) * (x[i] - centers[labels[i]]); if (d > fd) { fd = d; far = i; } }
      int ol = labels[far];
      ++fr[R_RELOC];
      centers_new[ol] -= x[far]; wsum[ol] -= 1.0;
      centers_new[j] = x[far]; wsum[j] = 1.0;
      x2[far] = x2[far]; /* labels are NOT updated by sklearn here */
    }
    acc_t shift_tot = 0.0;
    for (int j = 0; j < k; ++j) {
      double cn_j = (double)centers_new[j];
      if (wsum[j] > 0.0) cn_j = (double)(centers_new[j] * (1.0 / wsum[j]));
      double d = cn_j - centers[j]; d = fabs(d);
      shift_tot += d * d;
      centers[j] = cn_j;
    }
    fr[R_LLOYD_ITER] = it + 1;
    int same = 1;
    for (int i = 0; i < n; ++i) if (labels[i] != labels_old[i]) { same = 0; break; }
    if (same) { strict = 1; fr[R_LLOYD_STRICT] = 1; break; }
    if (shift_tot <= tol) break;
    memcpy(labels_old, labels, sizeof(int) * (size_t)n);
  }
  if (!strict) {
    double cn[TW_GMM_MAX_COMP];
    for (int j = 0; j < k; ++j) cn[j] = centers[j] * centers[j];
    for (int i = 0; i < n; ++i) labels[i] = nearest_centre(centers, cn, k, x[i], &fr[R_LLOYD_TIES]);
  }
}

/* ---- GaussianMixture ---------------------------------------------------------------------- */
/* weighted log prob of sample x under component c; `full` selects the covariance_type formula */
static double comp_logprob(const gmm_t* g, int c, double x, int full) {
  double lp;
  if (full) {
    double y = x * g->pc[c] - g->mu[c] * g->pc[c];
    lp = y * y;
  } else {
    double prec = g->pc[c] * g->pc[c];
    lp = (g->mu[c] * g->mu[c]) * prec - 2.0 * (x * (g->mu[c] * prec)) + (x * x) * prec;
  }
  return (-0.5 * (LOG_2PI + lp) + log(g->pc[c])) + log(g->w[c]);
}
static double lse(const double* a, int k) { /* scipy.special.logsumexp */
  double amax = -INFINITY; for (int c = 0; c < k; ++c) if (a[c] > amax) amax = a[c];
  acc_t s = 0.0; double m = 0.0;
  for (int c = 0; c < k; ++c) { if (a[c] == amax) m += 1.0; else s += exp(a[c] - amax); }
  if (s != 0.0) s /= m;
  return log1p((double)s) + log(m) + amax;
}
/* M-step / initialisation from responsibilities: returns -1 where sklearn raises ValueError */
static int m_step(gmm_t* g, const double* x, int n, const double* resp, int full, int init) {
  int k = g->k;
  double nk[TW_GMM_MAX_COMP];
  for (int c = 0; c < k; ++c) {
    acc_t s = 0.0; for (int i = 0; i < n; ++i) s += resp[(size_t)i * k + c];
    nk[c] = (double)s + 10.0 * DBL_EPS;
    acc_t sx = 0.0; for (int i = 0; i < n; ++i) sx += resp[(size_t)i * k + c] * x[i];
    g->mu[c] = (double)sx / nk[c];
    if (full) {
      acc_t sv = 0.0;
      for (int i = 0; i < n; ++i) { double d = x[i] - g->mu[c]; sv += (resp[(size_t)i * k + c] * d) * d; }
      g->cov[c] = (double)sv / nk[c] + REG_COVAR;
    } else {
      acc_t sx2 = 0.0; for (int i = 0; i < n; ++i) sx2 += resp[(size_t)i * k + c] * (x[i] * x[i]);
      g->cov[c] = (double)(sx2 / nk[c] - (acc_t)g->mu[c] * g->mu[c]) + REG_COVAR;
    }
    if (!(g->cov[c] > 0.0)) return -1;
    g->pc[c] = 1.0 / sqrt(g->cov[c]);
  }
  if (init) { for (int c = 0; c < k; ++c) g->w[c] = nk[c] / (double)n; }
  else { acc_t s = 0.0; for (int c = 0; c < k; ++c) s += nk[c]; for (int c = 0; c < k; ++c) g->w[c] = nk[c] / (double)s; }
  return 0;
}

static int gmm_fit(const double* x, int n, int k, int full, mt_t* rng, gmm_t* g, double* work /* 4n + n*k */,
                   int* labels, int32_t* fr) {
  memset(fr, 0, sizeof(fitrec_t));
  if (n < 2 || n < k) { /* sklearn: ensure_min_samples=2 / n_samples >= n_components */
    /* the k-means draw is never reached */
    fr[R_STATUS] = -1;
    return -1;
  }
  fr[R_STATUS] = -2;    /* ValueError from a non-positive covariance, unless the fit completes */
  g->k = k;
  kmeans_labels(x, n, k, rng, labels, work, fr);
  double* resp = work + 4 * (size_t)n;
  for (int i = 0; i < n; ++i) for (int c = 0; c < k; ++c) resp[(size_t)i * k + c] = labels[i] == c ? 1.0 : 0.0;
  if (m_step(g, x, n, resp, full, 1)) return -1;
  double lower = -INFINITY;
  g->converged = 0;
  double* lpn = work; /* reuse: n doubles */
  for (int it = 1; it <= EM_MAX_ITER; ++it) {
    double prev = lower;
    for (int i = 0; i < n; ++i) {
      double a[TW_GMM_MAX_COMP];
      for (int c = 0; c < k; ++c) a[c] = comp_logprob(g, c, x[i], full);
      double l = lse(a, k);
      lpn[i] = l;
      for (int c = 0; c < k; ++c) resp[(size_t)i * k + c] = exp(a[c] - l);
    }
    lower = pw_sum(lpn, n) / (double)n;
    fr[R_EM_ITER] = it;
    if (m_step(g, x, n, resp, full, 0)) return -1;
    g->n_iter = it;
    if (fabs(lower - prev) < EM_TOL) { g->converged = 1; break; }
  }
  fr[R_EM_CONVERGED] = g->converged;
  fr[R_STATUS] = 1;
  return 0;
}

static double gmm_score(const gmm_t* g, const double* x, int n, int full, double* work) {
  for (int i = 0; i < n; ++i) {
    double a[TW_GMM_MAX_COMP];
    for (int c = 0; c < g->k; ++c) a[c] = comp_logprob(g, c, x[i], full);
    work[i] = lse(a, g->k);
  }
  return pw_sum(work, n) / (double)n;
}

static int cmp_dbl(const void* a, const void* b) {
  double x = *(const double*)a, y = *(const double*)b;
  return x < y ? -1 : x > y;
}

/* draws of random_sample() consumed by the model-selection fits of one term */
int two_gmm_draws_for(int max_n) {
  int tot = 0;
  for (int k = 1; k <= max_n; ++k) tot += 1 + (k - 1) * (2 + (int)log((double)k));
  return tot;
}

/* One term: returns n_selected (0 = degenerate Gaussian record).  bic (may be NULL) gets the 'diag' BIC
 * of every K = 1..5, +inf where the fit is not tried or raises. */
static int refit_term(const double* x, int n, uint32_t seed_select, uint32_t rng_skip, double* rec,
                      int* max_n_out, double* bic_out, int32_t* rec_out) {
  fitrec_t frs[TW_GMM_MAX_COMP + 1];
  memset(frs, 0, sizeof frs);
  if (bic_out) for (int k = 0; k < TW_GMM_MAX_COMP; ++k) bic_out[k] = INFINITY;
  memset(rec, 0, sizeof(double) * TW_MIX_REC);
  if (n == 0) { /* services_times = (0, 0) -> std clamp 0.001 (V3:765-766, V1:130-131) */
    rec[0] = 0.0; rec[1] = 0.0; rec[2] = 0.001; rec[3] = log(0.001);
    *max_n_out = 0;
    if (rec_out) memcpy(rec_out, frs, sizeof frs);
    return 0;
  }
  double* work = (double*)malloc(sizeof(double) * ((size_t)n * (5 + TW_GMM_MAX_COMP)));
  int* labels = (int*)malloc(sizeof(int) * (size_t)n);
  double* srt = work + 4 * (size_t)n + (size_t)n * TW_GMM_MAX_COMP;
  memcpy(srt, x, sizeof(double) * (size_t)n);
  qsort(srt, (size_t)n, sizeof(double), cmp_dbl);
  int uniq = 1; for (int i = 1; i < n; ++i) if (srt[i] != srt[i - 1]) ++uniq;
  int max_n = uniq < TW_GMM_MAX_COMP ? uniq : TW_GMM_MAX_COMP;
  *max_n_out = max_n;
  mt_t rng; mt_seed(&rng, seed_select);
  for (uint32_t q = 0; q < rng_skip; ++q) (void)mt_random_sample(&rng);
  int best_k = 0; double best_bic = INFINITY;
  for (int k = 1; k <= max_n; ++k) {
    gmm_t g;
    if (gmm_fit(x, n, k, 0, &rng, &g, work, labels, frs[k - 1])) continue;
    double sc = gmm_score(&g, x, n, 0, work);
    double bic = -2.0 * sc * (double)n + (double)(3 * k - 1) * log((double)n);
    if (getenv("TWO_GMM_DEBUG")) fprintf(stderr, "two_gmm: n=%d k=%d bic=%.6f\n", n, k, bic);
    if (bic_out) bic_out[k - 1] = bic;
    if (bic < best_bic) { best_bic = bic; best_k = k; }
  }
  int ret = 0;
  if (best_k > 0) {
    mt_t r100; mt_seed(&r100, 100u);
    gmm_t g;
    if (gmm_fit(x, n, best_k, 1, &r100, &g, work, labels, frs[TW_GMM_MAX_COMP]) == 0) {
      rec[0] = (double)best_k;
      for (int c = 0; c < best_k; ++c) {
        rec[1 + c] = g.pc[c]; rec[6 + c] = g.mu[c] * g.pc[c];
        rec[11 + c] = log(g.pc[c]); rec[16 + c] = log(g.w[c]);
      }
      ret = best_k;
    }
  }
  if (ret == 0) { rec[0] = 0.0; rec[1] = 0.0; rec[2] = 0.001; rec[3] = log(0.001); }
  if (rec_out) memcpy(rec_out, frs, sizeof frs);
  free(work); free(labels);
  return ret;
}

/*
 * rng_skip[t]: random_sample() calls consumed from the `seed_select` stream before term t's
 * model-selection fits (the reference fits terms one after the other from one global stream;
 * NULL = every term starts at the seed).  max_n_out[t] (may be NULL) returns min(#unique, 5) so
 * the caller can chain the skips.
 */
int two_gmm_refit_ex(int32_t n_terms, const int64_t* term_sample_off, const double* delays,
                     const int32_t* counts, uint32_t seed_select, const uint32_t* rng_skip,
                     double* mix_out, int32_t* n_selected_out, int32_t* max_n_out) {
  return two_gmm_refit_record(n_terms, term_sample_off, delays, counts, seed_select, rng_skip, mix_out,
                              n_selected_out, max_n_out, NULL, NULL);
}

/* two_gmm_refit_ex and the decisions of every fit.  bic_out[t * 5 + k - 1]: the 'diag' BIC of term t with
 * k components (+inf where that fit is not tried or raises).  rec_out[(t * 6 + f) * 7 + field], f = k - 1
 * for the 'diag' fits and f = 5 for the final 'full' fit; fields: status (0 not tried, -1 too few samples,
 * -2 ValueError, 1 fitted), Lloyd iterations, Lloyd stopped on unchanged labels (1) or on the centre
 * shift (0), empty-cluster relocations, EM iterations, EM converged, first centre in the replay band, Lloyd
 * labels whose runner-up centre is within rounding (nearest_centre). */
int two_gmm_refit_record(int32_t n_terms, const int64_t* term_sample_off, const double* delays,
                         const int32_t* counts, uint32_t seed_select, const uint32_t* rng_skip,
                         double* mix_out, int32_t* n_selected_out, int32_t* max_n_out, double* bic_out,
                         int32_t* rec_out) {
  for (int t = 0; t < n_terms; ++t) {
    int mx = 0;
    int k = refit_term(delays + term_sample_off[t], counts[t], seed_select, rng_skip ? rng_skip[t] : 0u,
                       mix_out + (size_t)t * TW_MIX_REC, &mx, bic_out ? bic_out + (size_t)t * TW_GMM_MAX_COMP : NULL,
                       rec_out ? rec_out + (size_t)t * (TW_GMM_MAX_COMP + 1) * TW_GMM_REC_FIELDS : NULL);
    if (n_selected_out) n_selected_out[t] = k;
    if (max_n_out) max_n_out[t] = mx;
  }
  return TW_OK;
}

int two_gmm_refit(int32_t n_terms, const int64_t* term_sample_off, const double* delays,
                  const int32_t* counts, uint32_t seed_select, double* mix_out, int32_t* n_selected_out) {
  return two_gmm_refit_ex(n_terms, term_sample_off, delays, counts, seed_select, NULL, mix_out, n_selected_out,
                          NULL);
}

/* debug / test hook: the k-means labels a fit with k components starts from, with the random stream
 * `seed` advanced by `skip` random_sample() draws (tests/test_oracle_gmm.py) */
int two_debug_kmeans_labels(const double* x, int n, int k, uint32_t seed, uint32_t skip, int* labels) {
  double* work = (double*)malloc(sizeof(double) * (size_t)n * 4);
  mt_t rng; mt_seed(&rng, seed);
  for (uint32_t q = 0; q < skip; ++q) (void)mt_random_sample(&rng);
  fitrec_t fr;
  memset(fr, 0, sizeof fr);
  kmeans_labels(x, n, k, &rng, labels, work, fr);
  free(work);
  return 0;
}
