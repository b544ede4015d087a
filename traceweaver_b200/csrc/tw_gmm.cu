// tw_gmm.cu — pass-boundary refit on the device: per score term a 1-D Gaussian mixture with
// 1..min(5, #unique) components, BIC model selection ('diag' fits), final 'full' fit.
//
// Replaces ComputeEpPairDistParams5's fitting half, traceweaver_v3.py:764-786, i.e. the calls
//     mixture.GaussianMixture(n_components=n, covariance_type='diag').fit(durations)   (x max_n)
//     mixture.GaussianMixture(n_components=n_selected, random_state=100).fit(durations)
// whose algorithm is scikit-learn's (k-means++ seeding + Lloyd for the initial responsibilities,
// EM until |delta lower bound| < 1e-3, reg_covar 1e-6, n_init 1, max_iter 100), driven by
// NumPy's legacy MT19937 stream.  The random_sample() values are data independent, so the host
// generates the stream once (tw_api.cu) and the kernels index it.  Discrete decisions (seeding
// draws, label assignment, stopping tests, BIC arg-min) follow the library's rules; sums are
// warp-parallel, so parameters agree with scikit-learn to ~1e-12 relative, not bit for bit.
//
// Mapping: ONE WARP PER FIT, no block barriers.  A fit never stores responsibilities: each EM
// iteration is a single sweep over the samples (32 per lane for n = 1000) that evaluates the
// E-step and accumulates the M-step's sufficient statistics (sum r, sum r x, sum r x^2 per
// component) in registers, reduced with shuffles.  k-means keeps no label / distance arrays
// either: labels and closest-centre distances are recomputed from the <= 5 centres.
//   k_gmm_prep  : warp per term      -> min(#unique, 5), mean, variance
//   k_gmm_skip  : thread per problem -> position of every term in the model-selection stream
//   k_gmm_bic   : warp per (term, k) -> BIC of the 'diag' fit with k components
//   k_gmm_final : warp per term      -> arg-min BIC, 'full' fit, TW_MIX_REC record
#include "tw_kernels.cuh"

namespace tw {

constexpr double kRegCovar = 1e-6;
constexpr double kEmTol = 1e-3;
constexpr int kEmMaxIter = 100;
constexpr int kKmMaxIter = 300;
constexpr double kKmTol = 1e-4;
constexpr double kDblEps = 2.220446049250313e-16;
constexpr int KC = TW_GMM_MAX_COMP;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kLloydLabelN = 1024;   // longest sample list whose Lloyd labels stay in shared memory

// phase counters (tw_kernels.cuh): cycles in seeding / Lloyd / initial M-step / EM / scoring in 0-4,
// then Lloyd iterations, EM iterations and fits in 5-7
TW_PHASE_BANK(g_gmm_phase);
#ifdef TW_PROFILE_PHASES
cudaError_t gmm_phase_bank(void** bank) { return cudaGetSymbolAddress(bank, g_gmm_phase); }
#endif

// Work of the EM sweeps (always on; one atomic per fit): sample-component evaluations of the E+M sweep.
// bench.py turns it into the FP64 roofline of the refit (tw_gmm_work, include/traceweaver_b200.h).
__device__ unsigned long long g_gmm_em_evals;

__device__ __forceinline__ double wsum(double v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(kFull, v, d);
  return v;
}

// n_local_trials = 2 + int(ln k) of sklearn's k-means++: 2, 2, 3, 3, 3 for k = 1..5
__device__ __forceinline__ int trials_for_k(int k) { return k < 3 ? 2 : 3; }
__device__ __forceinline__ int draws_for_k(int k) { return 1 + (k - 1) * trials_for_k(k); }

// _euclidean_distances(squared=True): -2 c x + c^2 + x^2, clipped at 0.  The product by -2 is exact,
// so the fused form rounds the same sum as dadd(dmul(-2.0, dmul(c, x)), c2).
__device__ __forceinline__ double sq_dist(double c, double c2, double x, double x2) {
  double d = dadd(__fma_rn(-2.0, dmul(c, x), c2), x2);
  return d > 0.0 ? d : 0.0;
}

// A fit's parameters.  They are the same on every lane, so each warp keeps them in a shared-memory
// slot (the E-step reads them as broadcasts) instead of 4K registers per thread.
struct Fit {
  double mu[KC], pc[KC], logpc[KC], logw[KC];
};

// arg-min over centres of c^2 - 2 x c (the x^2 term is common), first minimum wins — evaluated as a
// tree (depth 3 for K = 5) instead of a chain; strict "<" with the lower index on the left keeps
// NumPy's tie rule.  cen2[j] = dmul(cen[j], cen[j]), computed once per set of centres; the product
// by -2 is exact, so the fused form rounds the same sum as dadd(cen2[j], dmul(-2.0, dmul(x, cen[j]))).
struct Near { double d; int j; };
__device__ __forceinline__ Near near_min(Near a, Near b) { return b.d < a.d ? b : a; }
template <int K>
__device__ __forceinline__ void centre_squares(const double* cen, double* cen2) {
#pragma unroll
  for (int j = 0; j < KC; ++j) cen2[j] = j < K ? dmul(cen[j], cen[j]) : 0.0;
}
template <int K>
__device__ __forceinline__ int nearest(const double* cen, const double* cen2, double x) {
  Near v[KC];
#pragma unroll
  for (int j = 0; j < KC; ++j) {
    v[j].j = j;
    v[j].d = j < K ? __fma_rn(-2.0, dmul(x, cen[j]), cen2[j]) : 0.0;
  }
  if (K == 1) return 0;
  if (K == 2) return near_min(v[0], v[1]).j;
  if (K == 3) return near_min(near_min(v[0], v[1]), v[2]).j;
  if (K == 4) return near_min(near_min(v[0], v[1]), near_min(v[2], v[3])).j;
  return near_min(near_min(near_min(v[0], v[1]), near_min(v[2], v[3])), v[4]).j;
}

// One lane's samples (i = lane, lane + 32, ...) two at a time, next pair loaded before the current
// one is processed: f(x0, x1, valid1, s) with s the lane-local index of x0.  The two samples are
// independent until the accumulators, which gives the FP64 pipe two chains to interleave; f must
// add x0's contribution before x1's so that every lane sums in the same order as a plain loop.
template <class F>
__device__ __forceinline__ void sweep2(const double* __restrict__ x, int n, F&& f) {
  int i = threadIdx.x & 31;
  double a = i < n ? x[i] : 0.0;
  double b = i + 32 < n ? x[i + 32] : 0.0;
  for (int s = 0; i < n; i += 64, s += 2) {
    const double x0 = a, x1 = b;
    const bool v1 = i + 32 < n;
    a = i + 64 < n ? x[i + 64] : 0.0;
    b = i + 96 < n ? x[i + 96] : 0.0;
    f(x0, x1, v1, s);
  }
}

// k-means++ seeding of KMeans(n_clusters=K, n_init=1).fit(X) on centred data (x - mean).
// draws[] = this fit's random_sample() values.
template <int K>
__device__ __forceinline__ void seed_centres(const double* __restrict__ x, int n, double mean,
                                             const double* __restrict__ draws, double* cen) {
  const int lane = threadIdx.x & 31;
  const int k = K;
  TW_PHASE_START(phase_t0);
#pragma unroll
  for (int j = 0; j < KC; ++j) cen[j] = 0.0;
  // ---- k-means++ seeding.  First centre: RandomState.choice(n, p=1/n) (first_centre, tw_core.cuh).
  cen[0] = dsub(x[first_centre(draws[0], n)], mean);
  const int trials = trials_for_k(k);
  double pot = 0.0;
  {
    double part = 0.0, c2 = dmul(cen[0], cen[0]);
    for (int i = lane; i < n; i += 32) { double xi = dsub(x[i], mean); part = dadd(part, sq_dist(cen[0], c2, xi, dmul(xi, xi))); }
    pot = wsum(part);
  }
  for (int ci = 1; ci < k; ++ci) {
    double rv[3];
    int cand[3];
    for (int t = 0; t < 3; ++t) { rv[t] = t < trials ? dmul(draws[1 + (ci - 1) * trials + t], pot) : 0.0; cand[t] = n - 1; }
    bool found[3] = {false, false, false};
    // np.searchsorted(np.cumsum(closest), rv): first i with cumsum_i >= rv, rounds of 32 samples
    double carry = 0.0;
    for (int base = 0; base < n; base += 32) {
      int i = base + lane;
      double cl = 0.0;
      if (i < n) {
        double xi = dsub(x[i], mean), x2 = dmul(xi, xi);
        cl = sq_dist(cen[0], dmul(cen[0], cen[0]), xi, x2);
        for (int j = 1; j < ci; ++j) { double d = sq_dist(cen[j], dmul(cen[j], cen[j]), xi, x2); cl = d < cl ? d : cl; }
      }
      double incl = cl;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        double o = __shfl_up_sync(kFull, incl, d);
        if (lane >= d) incl = dadd(incl, o);
      }
      incl = dadd(incl, carry);
      for (int t = 0; t < trials; ++t) {
        if (found[t]) continue;
        unsigned m = __ballot_sync(kFull, i < n && incl >= rv[t]);
        if (m) { cand[t] = base + __ffs(m) - 1; found[t] = true; }
      }
      carry = __shfl_sync(kFull, incl, 31);
      if (found[0] && (trials < 2 || found[1]) && (trials < 3 || found[2])) break;
    }
    double cc[3], part[3] = {0.0, 0.0, 0.0};
    for (int t = 0; t < 3; ++t) cc[t] = dsub(x[cand[t]], mean);
    for (int i = lane; i < n; i += 32) {
      double xi = dsub(x[i], mean), x2 = dmul(xi, xi);
      double cl = sq_dist(cen[0], dmul(cen[0], cen[0]), xi, x2);
      for (int j = 1; j < ci; ++j) { double d = sq_dist(cen[j], dmul(cen[j], cen[j]), xi, x2); cl = d < cl ? d : cl; }
      for (int t = 0; t < trials; ++t) {
        double d = sq_dist(cc[t], dmul(cc[t], cc[t]), xi, x2);
        part[t] = dadd(part[t], d < cl ? d : cl);
      }
    }
    int best = 0;
    double bp = wsum(part[0]);
    for (int t = 1; t < trials; ++t) {
      double pt = wsum(part[t]);
      if (pt < bp) { bp = pt; best = t; }
    }
    cen[ci] = cc[best];
    pot = bp;
  }
  TW_PHASE(g_gmm_phase, phase_t0, 0);
}

// Lloyd iterations from the seeded centres: cen[] in, the centres that define the final labels_ out.
// labs = this warp's kLloydLabelN bytes of shared memory.
template <int K>
__device__ __forceinline__ void lloyd_centres(const double* __restrict__ x, int n, double mean, double tol,
                                              const double* cen_in, double* cen_out, unsigned char* labs) {
  const int lane = threadIdx.x & 31;
  const int k = K;
  TW_PHASE_START(phase_t0);
  double cen[KC];
#pragma unroll
  for (int j = 0; j < KC; ++j) cen[j] = cen_in[j];
  // ---- Lloyd (_kmeans_single_lloyd).  The labels of the previous assignment (needed for the
  // "no label changed" stop) live in one shared-memory byte per sample when n <= kLloydLabelN;
  // sample i is only ever read and written by lane i % 32.  Longer sample lists recompute them from
  // the previous centres.  With at most 32 samples per lane, a lane's K counts fit in 6-bit fields
  // of one word.
  double prev[KC], cen2[KC];
#pragma unroll
  for (int j = 0; j < KC; ++j) prev[j] = cen[j];
  bool have_prev = false, strict = false;
  const bool packed = n <= kLloydLabelN;
  for (int it = 0; it < kKmMaxIter; ++it) {
    double sx[KC];
    int cnt_i[KC];
#pragma unroll
    for (int j = 0; j < KC; ++j) { sx[j] = 0.0; cnt_i[j] = 0; }
    bool changed = !have_prev;
    centre_squares<K>(cen, cen2);
    if (packed) {
      unsigned cnt_p = 0u;
      sweep2(x, n, [&](double x0, double x1, bool v1, int s) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const double xi = dsub(h ? x1 : x0, mean);
          const bool valid = h ? v1 : true;
          const int lab = nearest<K>(cen, cen2, xi);
          if (valid) {
            unsigned char& old = labs[lane + 32 * (s + h)];
            changed |= have_prev && old != lab;                     // first sweep: forced true below
            old = (unsigned char)lab;
            cnt_p += 1u << (6 * lab);
          }
#pragma unroll
          for (int j = 0; j < K; ++j) sx[j] = dadd(sx[j], valid && j == lab ? xi : 0.0);
        }
      });
#pragma unroll
      for (int j = 0; j < K; ++j) cnt_i[j] = (int)((cnt_p >> (6 * j)) & 63u);
    } else {
      double prev2[KC];
      centre_squares<K>(prev, prev2);
      for (int i = lane; i < n; i += 32) {
        const double xi = dsub(x[i], mean);
        const int lab = nearest<K>(cen, cen2, xi);
        if (have_prev && nearest<K>(prev, prev2, xi) != lab) changed = true;
#pragma unroll
        for (int j = 0; j < K; ++j) {
          const bool m = j == lab;
          sx[j] = dadd(sx[j], m ? xi : 0.0);
          cnt_i[j] += m ? 1 : 0;
        }
      }
    }
    if (!have_prev) changed = true;
    // the K count reductions, the K sum butterflies (each in wsum's order) and the vote are
    // independent: issued together, their latencies overlap
    double cnt[KC];
#pragma unroll
    for (int j = 0; j < KC; ++j) cnt[j] = j < K ? (double)__reduce_add_sync(kFull, cnt_i[j]) : 0.0;
    changed = __any_sync(kFull, changed);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
#pragma unroll
      for (int j = 0; j < K; ++j) sx[j] += __shfl_xor_sync(kFull, sx[j], d);
    }
    // _relocate_empty_clusters_dense (rare): farthest point from its centre moves to the empty cluster
    for (int j = 0; j < k; ++j) {
      bool empty = false;          // cnt[j] == 0, selected without indexing cnt[] by a run-time j
#pragma unroll
      for (int q = 0; q < K; ++q) empty = q == j ? cnt[q] == 0.0 : empty;
      if (!empty) continue;
      double fd = -1.0;
      int fi = 0x7fffffff;
      for (int i = lane; i < n; i += 32) {
        double xi = dsub(x[i], mean);
        const int nl = nearest<K>(cen, cen2, xi);
        double cn = cen[0];
#pragma unroll
        for (int q = 1; q < KC; ++q) cn = q == nl ? cen[q] : cn;
        double d = dsub(xi, cn);
        d = dmul(d, d);
        if (d > fd) { fd = d; fi = i; }
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        double od = __shfl_xor_sync(kFull, fd, d);
        int oi = __shfl_xor_sync(kFull, fi, d);
        if (od > fd || (od == fd && oi < fi)) { fd = od; fi = oi; }
      }
      double xf = dsub(x[fi], mean);
      int ol = nearest<K>(cen, cen2, xf);
#pragma unroll
      for (int q = 0; q < KC; ++q) {
        if (q == ol) { sx[q] = dsub(sx[q], xf); cnt[q] -= 1.0; }
        if (q == j) { sx[q] = xf; cnt[q] = 1.0; }
      }
    }
    double shift_tot = 0.0;
#pragma unroll
    for (int j = 0; j < KC; ++j) {
      prev[j] = cen[j];
      if (j < k) {
        double nc = cnt[j] > 0.0 ? dmul(sx[j], 1.0 / cnt[j]) : sx[j];
        double d = fabs(dsub(nc, cen[j]));
        shift_tot = __fma_rn(d, d, shift_tot);
        cen[j] = nc;
      }
    }
    have_prev = true;
    TW_COUNT(g_gmm_phase, 5, 1);
    if (!changed) { strict = true; break; }
    if (shift_tot <= tol) break;
  }
  // strict convergence keeps the labels of the last assignment (w.r.t. the centres before the
  // final update); otherwise sklearn re-runs the assignment with the final centres
#pragma unroll
  for (int j = 0; j < KC; ++j) cen_out[j] = strict ? prev[j] : cen[j];
  TW_PHASE(g_gmm_phase, phase_t0, 1);
}

// v[lane] on lanes 0..K-1, v[0] on the others: hands each of the first K lanes its component of a
// warp-uniform per-component array
template <int K>
__device__ __forceinline__ double lane_component(const double* v) {
  const int lane = threadIdx.x & 31;
  double r = v[0];
#pragma unroll
  for (int c = 1; c < K; ++c) r = lane == c ? v[c] : r;
  return r;
}

// parameters from the M-step sums, component c on lane c (lanes >= K idle), written to the warp's
// shared slot f; the arguments are lane c's component.  nk = sum r, mup = sum r x' / nk
// (x' = x - shift), tot = nk summed over the components in order c = 0..K-1.
//   'diag': S2 = sum r x^2 with shift = 0 and cov = S2/nk - mu^2 + reg — scikit-learn's own
//           avg_X2 - means^2 formula (_estimate_gaussian_covariances_diag);
//   'full': S2 = sum r (x' - mu')^2 from a second sweep (_estimate_gaussian_covariances_full),
//           so a component of identical samples gets cov = reg_covar exactly, as in the library.
// The roundings are spelled out so that the fits keep the bits they had when every lane evaluated
// every component with the plain expressions: there -O3 contracted component 0's S2/nk - mup^2 into
// one fused multiply-add and left the other components' product and difference separately rounded.
// The 'diag' BIC arg-min is ill-conditioned on terms with few distinct delays, so one ulp of one
// covariance can move the selected K (tests/gmm_conditioning.py).
template <int K, bool FULL>
__device__ __forceinline__ bool params_from_stats(Fit& f, int n, double nk, double mup, double S2, double tot,
                                                  double shift, bool init) {
  const int c = threadIdx.x & 31;
  bool ok = true;
  __syncwarp();                      // the E-step reads of the previous parameters are done
  if (c < K) {
    const double q = __ddiv_rn(S2, nk);
    const double cov = FULL     ? __dadd_rn(q, kRegCovar)
                       : c == 0 ? __dadd_rn(fma(-mup, mup, q), kRegCovar)
                                : __dadd_rn(__dsub_rn(q, __dmul_rn(mup, mup)), kRegCovar);
    ok = cov > 0.0;
    const double pc = __ddiv_rn(1.0, sqrt(cov));
    f.mu[c] = __dadd_rn(mup, shift);
    f.pc[c] = pc;
    f.logpc[c] = log(pc);
    f.logw[c] = log(__ddiv_rn(nk, init ? (double)n : tot));
  }
  __syncwarp();
  return __all_sync(kFull, ok);
}

// E-step of one sample.  a[c] <- exp(w_c - max w) with w_c the weighted log-probabilities (sklearn
// _estimate_log_gaussian_prob + log weights, same operation order); returns their sum t >= 1, so
// that logsumexp = *amax + log t and the responsibilities are a[c] / t.
template <int K, bool FULL>
__device__ __forceinline__ double estep(const Fit& f, const double* __restrict__ tab, double x, double* a,
                                        double* amax_out) {
  double amax = -INFINITY;
#pragma unroll
  for (int c = 0; c < K; ++c) {
    double lp;
    if (FULL) {
      double y = dsub(dmul(x, f.pc[c]), dmul(f.mu[c], f.pc[c]));
      lp = dmul(y, y);
    } else {
      double prec = dmul(f.pc[c], f.pc[c]);
      lp = dadd(dsub(dmul(dmul(f.mu[c], f.mu[c]), prec), dmul(2.0, dmul(x, dmul(f.mu[c], prec)))),
                dmul(dmul(x, x), prec));
    }
    a[c] = dadd(dadd(dmul(-0.5, dadd(TW_LOG_2PI, lp)), f.logpc[c]), f.logw[c]);
    amax = a[c] > amax ? a[c] : amax;
  }
  double t = 0.0;
#pragma unroll
  for (int c = 0; c < K; ++c) {
    // exp(d) < 2^-57 for d < -40: it cannot change a sum that holds the maximum's 1.0
    const double d = a[c] - amax;
    const double e = exp_neg(tab, d);
    a[c] = d >= -40.0 ? e : 0.0;
    t += a[c];
  }
  *amax_out = amax;
  return t;
}

// running sum of logsumexp values: sum(amax) + log(prod t), the product flushed before it can overflow
struct LogSum {
  double acc = 0.0, prod = 1.0;
  int cnt = 0;
  __device__ __forceinline__ void add(double t, double amax) {
    acc += amax;
    prod *= t;                       // 1 <= t <= 5
    if (++cnt == 128) { acc += log(prod); prod = 1.0; cnt = 0; }
  }
  __device__ __forceinline__ double total() const { return acc + log(prod); }
};

// GaussianMixture(K, covariance_type = FULL ? 'full' : 'diag').fit(x) by one warp.
// Returns false on scikit-learn's ValueError paths; *score = mean log-likelihood under the final
// parameters when want_score.
// The k-means initialisation arrives as its label centres `cen` (k_gmm_seed / k_gmm_lloyd).
template <int K, bool FULL>
__device__ __forceinline__ bool em_fit(const double* __restrict__ x, int n, double mean, const double* cen,
                                       const double* __restrict__ tab, Fit& f, bool want_score, double* score) {
  const int lane = threadIdx.x & 31;
  const int k = K;
  if (n < 2 || n < k) return false;
  const double shift = FULL ? mean : 0.0;
  double S0[KC], S1[KC], S2[KC], nk[KC], mup[KC];
  double my_nk, my_mup, my_s2;       // this lane's component (lanes 0..K-1)
  TW_PHASE_START(phase_t0);
  {
    double cen2[KC];
    centre_squares<K>(cen, cen2);
    TW_COUNT(g_gmm_phase, 7, 1);
#pragma unroll
    for (int c = 0; c < KC; ++c) { S0[c] = 0.0; S1[c] = 0.0; S2[c] = 0.0; }
    sweep2(x, n, [&](double x0, double x1, bool v1, int) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const double xi = h ? x1 : x0;
        const int lab = (h ? v1 : true) ? nearest<K>(cen, cen2, xi - mean) : -1;
        const double xs = xi - shift, xs2 = xs * xs;
#pragma unroll
        for (int c = 0; c < K; ++c) {
          const bool m = c == lab;
          S0[c] += m ? 1.0 : 0.0;
          S1[c] += m ? xs : 0.0;
          S2[c] += m ? xs2 : 0.0;
        }
      }
    });
#pragma unroll
    for (int c = 0; c < K; ++c) {
      nk[c] = wsum(S0[c]) + 10.0 * kDblEps;
      S1[c] = wsum(S1[c]);
      S2[c] = wsum(S2[c]);
    }
    my_nk = lane_component<K>(nk);
    my_mup = __ddiv_rn(lane_component<K>(S1), my_nk);
    if (FULL) {   // second sweep: sum of squared deviations from the new means
#pragma unroll
      for (int c = 0; c < K; ++c) mup[c] = __shfl_sync(kFull, my_mup, c);
#pragma unroll
      for (int c = 0; c < KC; ++c) S2[c] = 0.0;
      sweep2(x, n, [&](double x0, double x1, bool v1, int) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const double xi = h ? x1 : x0;
          const int lab = (h ? v1 : true) ? nearest<K>(cen, cen2, xi - mean) : -1;
          const double xs = xi - shift;
#pragma unroll
          for (int c = 0; c < K; ++c) {
            const double d = xs - mup[c];
            S2[c] += c == lab ? d * d : 0.0;
          }
        }
      });
#pragma unroll
      for (int c = 0; c < K; ++c) S2[c] = wsum(S2[c]);
    }
    my_s2 = lane_component<K>(S2);
  }
  if (!params_from_stats<K, FULL>(f, n, my_nk, my_mup, my_s2, 0.0, shift, true)) return false;
  TW_PHASE(g_gmm_phase, phase_t0, 2);
  double lower = -INFINITY;
  int em_sweeps = 0;
  for (int it = 1; it <= kEmMaxIter; ++it) {
    const double prev = lower;
    LogSum ls;
#pragma unroll
    for (int c = 0; c < KC; ++c) { S0[c] = 0.0; S1[c] = 0.0; S2[c] = 0.0; }
    for (int i = lane; i < n; i += 32) {
      double xi = x[i], a[KC], amax;
      const double t = estep<K, FULL>(f, tab, xi, a, &amax);
      ls.add(t, amax);
      const double inv = 1.0 / t;
#pragma unroll
      for (int c = 0; c < K; ++c) {
        const double r = a[c] * inv;
        S0[c] += r;
        if (FULL) {
          // deviations from the OLD mean: sum r (x - mu_new)^2 = S2 - (S1 / S0) S1 below.  Near
          // convergence mu_new ~ mu_old, so nothing cancels, and a component of identical samples
          // still gets cov = reg_covar (to ~1e-30) as in _estimate_gaussian_covariances_full.
          const double dx = xi - f.mu[c];
          const double rd = r * dx;
          S1[c] += rd;
          S2[c] += rd * dx;
        } else {
          S1[c] += r * xi;
          S2[c] += r * (xi * xi);
        }
      }
    }
    lower = wsum(ls.total()) / (double)n;
    double tot = 0.0;
#pragma unroll
    for (int c = 0; c < K; ++c) {
      nk[c] = wsum(S0[c]) + 10.0 * kDblEps;
      tot += nk[c];
      S1[c] = wsum(S1[c]);
      S2[c] = wsum(S2[c]);
    }
    my_nk = lane_component<K>(nk);
    const double s1 = lane_component<K>(S1);
    my_s2 = lane_component<K>(S2);
    if (FULL) {      // S2 - delta s1 is one fused multiply-add, as -O3 contracted it before
      const double delta = __ddiv_rn(s1, my_nk);
      my_s2 = fma(-delta, s1, my_s2);
      if (my_s2 < 0.0) my_s2 = 0.0;
      my_mup = __dsub_rn(__dadd_rn(f.mu[lane < K ? lane : 0], delta), shift);
    } else {
      my_mup = __ddiv_rn(s1, my_nk);
    }
    if (!params_from_stats<K, FULL>(f, n, my_nk, my_mup, my_s2, tot, shift, false)) {
      if (lane == 0) atomicAdd(&g_gmm_em_evals, (unsigned long long)it * (unsigned long long)n * K);
      return false;
    }
    TW_COUNT(g_gmm_phase, 6, 1);
    em_sweeps = it;
    if (fabs(lower - prev) < kEmTol) break;
  }
  if (lane == 0) atomicAdd(&g_gmm_em_evals, (unsigned long long)(em_sweeps + (want_score ? 1 : 0)) * (unsigned long long)n * K);
  TW_PHASE(g_gmm_phase, phase_t0, 3);
  if (want_score) {
    LogSum ls;
    for (int i = lane; i < n; i += 32) {
      double a[KC], amax;
      const double t = estep<K, FULL>(f, tab, x[i], a, &amax);
      ls.add(t, amax);
    }
    *score = wsum(ls.total()) / (double)n;
  }
  TW_PHASE(g_gmm_phase, phase_t0, 4);
  return true;
}

// ---------------------------------------------------------------------------------------------
// per-term statistics: min(#unique, 5) (V3:768), mean, variance
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_gmm_prep(int n_terms, const int64_t* __restrict__ term_sample_off, const double* __restrict__ delays,
           const int32_t* __restrict__ counts, int32_t* __restrict__ max_n, double* __restrict__ mean_var) {
  const int t = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= n_terms) return;
  const double* x = delays + term_sample_off[t];
  const int n = counts[t];
  double set[KC];
  int ns = 0;
  double part = 0.0;
  for (int i = lane; i < n; i += 32) {
    double v = x[i];
    part += v;
    bool seen = false;
#pragma unroll
    for (int q = 0; q < KC; ++q)
      if (q < ns && set[q] == v) seen = true;
    if (!seen && ns < KC) {
#pragma unroll
      for (int q = 0; q < KC; ++q)
        if (q == ns) set[q] = v;
      ++ns;
    }
  }
  // merge the lanes' small sets on lane 0's view (all lanes run the same merge)
  double mset[KC];
  int mn = 0;
  for (int src = 0; src < 32 && mn < KC; ++src) {
    int sn = __shfl_sync(kFull, ns, src);
    for (int q = 0; q < KC; ++q) {
      double v = __shfl_sync(kFull, set[q < KC ? q : 0], src);
      if (q >= sn || mn >= KC) continue;
      bool seen = false;
#pragma unroll
      for (int r = 0; r < KC; ++r)
        if (r < mn && mset[r] == v) seen = true;
      if (!seen) {
#pragma unroll
        for (int r = 0; r < KC; ++r)
          if (r == mn) mset[r] = v;
        ++mn;
      }
    }
  }
  double mean = n > 0 ? wsum(part) / (double)n : 0.0;
  double p2 = 0.0;
  for (int i = lane; i < n; i += 32) { double d = x[i] - mean; p2 += d * d; }
  double var = n > 0 ? wsum(p2) / (double)n : 0.0;
  if (lane == 0) {
    max_n[t] = n > 0 ? mn : 0;
    mean_var[2 * t] = mean;
    mean_var[2 * t + 1] = var;
  }
}

// position of every term in the model-selection random stream: the reference fits the terms of a
// service one after the other (order = term_rank) from ONE stream, after the fits on the true
// assignments (prob_base_skip[p] draws, 0 when there is no truth pass).
__global__ void k_gmm_skip(int n_problems, const int32_t* __restrict__ prob_ep_off,
                           const int32_t* __restrict__ ep_term_off, const int32_t* __restrict__ term_order,
                           const int32_t* __restrict__ max_n, const uint32_t* __restrict__ prob_base_skip,
                           uint32_t* __restrict__ rng_skip) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_problems) return;
  int t0 = ep_term_off[prob_ep_off[p]], t1 = ep_term_off[prob_ep_off[p + 1]];
  uint32_t pos = prob_base_skip ? prob_base_skip[p] : 0u;
  for (int q = t0; q < t1; ++q) {
    int t = term_order ? term_order[q] : q;   // global term index visited q-th
    rng_skip[t] = pos;
    int mn = max_n[t];
    for (int k = 1; k <= mn; ++k) pos += (uint32_t)draws_for_k(k);
  }
}

// draws the model-selection fits of each problem consume (truth pass bookkeeping)
__global__ void k_gmm_draws(int n_problems, const int32_t* __restrict__ prob_ep_off,
                            const int32_t* __restrict__ ep_term_off, const int32_t* __restrict__ max_n,
                            uint32_t* __restrict__ prob_draws) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_problems) return;
  uint32_t pos = 0;
  for (int t = ep_term_off[prob_ep_off[p]]; t < ep_term_off[prob_ep_off[p + 1]]; ++t)
    for (int k = 1; k <= max_n[t]; ++k) pos += (uint32_t)draws_for_k(k);
  prob_draws[p] = pos;
}

// One kernel instance per component count K and per phase of the fit (seeding / Lloyd / EM): with K
// a compile-time constant every `c < k` test and component loop folds away and registers hold
// exactly K components; with the phases in separate launches every warp of an SM loops over the same
// few hundred instructions.  The fused single-kernel fit of the first versions (10 k SASS
// instructions for K = 5, warps spread over three different hot loops) lost issue slots to
// instruction fetch (stall_no_inst).
// Blocks of 128 threads per SM that the EM kernels are compiled for: 4 (16 warps) for K = 4, 5, whose
// register footprint would otherwise allow only 3; the smaller K reach 16 warps unconstrained.
constexpr int em_min_blocks(int K) { return K >= 4 ? 4 : 1; }
// Blocks per SM that the Lloyd kernels are compiled for: 12, 8, 8, 7, 6 for K = 1..5 (at most 40, 64,
// 64, 72, 80 registers, no spills).
constexpr int lloyd_min_blocks(int K) { return K == 1 ? 12 : K == 2 ? 8 : K == 3 ? 8 : K == 4 ? 7 : 6; }

// Which fit a warp works on.  Model selection (list == nullptr): warp w -> term w, active iff the
// reference tries K components for it (K <= min(#unique, 5)), draws at the term's stream position.
// Final fits (list != nullptr): warp w -> w-th term of the group whose BIC arg-min is K, draws from
// the random_state=100 stream.
struct FitSel {
  const int32_t* list;
  const uint32_t* hist;
  const int32_t* max_n;
  const uint32_t* rng_skip;
  const double* stream;
  int stream_len;
  int n_terms;
};

template <int K>
__device__ __forceinline__ bool select_fit(const FitSel& sel, const int32_t* __restrict__ counts, int* t_out,
                                           const double** draws_out, int* err_flag) {
  const unsigned w = (blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5;
  int t;
  const double* draws;
  if (sel.list) {
    if (w >= sel.hist[K]) return false;
    uint32_t off = 0;
#pragma unroll
    for (int q = 1; q < K; ++q) off += sel.hist[q];
    t = sel.list[off + w];
    draws = sel.stream;
  } else {
    if (w >= (unsigned)sel.n_terms) return false;
    t = (int)w;
    if (K > sel.max_n[t]) return false;
    uint32_t pos = sel.rng_skip[t];
#pragma unroll
    for (int q = 1; q < K; ++q) pos += (uint32_t)draws_for_k(q);
    if ((int)pos + draws_for_k(K) > sel.stream_len) {
      if (err_flag && (threadIdx.x & 31) == 0) atomicMin(err_flag, (int)TW_ERR_RANGE_LIMIT);
      return false;
    }
    draws = sel.stream + pos;
  }
  const int n = counts[t];
  if (n < 2 || n < K) return false;      // scikit-learn raises: the fit is skipped (BIC stays +inf)
  *t_out = t;
  *draws_out = draws;
  return true;
}

template <int K>
__global__ void __launch_bounds__(128)
k_gmm_seed(FitSel sel, const int64_t* __restrict__ term_sample_off, const double* __restrict__ delays,
           const int32_t* __restrict__ counts, const double* __restrict__ mean_var, double* __restrict__ cen_out,
           int* __restrict__ err_flag) {
  int t;
  const double* draws;
  if (!select_fit<K>(sel, counts, &t, &draws, err_flag)) return;   // flags a stream overrun for every K
  // A 1-component fit labels every sample 0 whatever the centre (nearest<1>), so em_fit never reads
  // the k-means result of K = 1: its seeding and Lloyd kernels have nothing more to do.
  if (K == 1) return;
  double cen[KC];
  seed_centres<K>(delays + term_sample_off[t], counts[t], mean_var[2 * t], draws, cen);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int j = 0; j < K; ++j) cen_out[(size_t)t * KC + j] = cen[j];
  }
}

template <int K>
__global__ void __launch_bounds__(128, lloyd_min_blocks(K))
k_gmm_lloyd(FitSel sel, const int64_t* __restrict__ term_sample_off, const double* __restrict__ delays,
            const int32_t* __restrict__ counts, const double* __restrict__ mean_var, double* __restrict__ cen_io) {
  if (K == 1) return;                    // see k_gmm_seed
  int t;
  const double* draws;
  if (!select_fit<K>(sel, counts, &t, &draws, nullptr)) return;
  __shared__ unsigned char labs[128 / 32 * kLloydLabelN];
  double cen[KC], out[KC];
#pragma unroll
  for (int j = 0; j < KC; ++j) cen[j] = j < K ? cen_io[(size_t)t * KC + j] : 0.0;
  lloyd_centres<K>(delays + term_sample_off[t], counts[t], mean_var[2 * t], mean_var[2 * t + 1] * kKmTol, cen, out,
                   labs + (threadIdx.x >> 5) * kLloydLabelN);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int j = 0; j < K; ++j) cen_io[(size_t)t * KC + j] = out[j];
  }
}

// 'diag' fit + BIC of the terms that try K components
template <int K>
__global__ void __launch_bounds__(128, em_min_blocks(K))
k_gmm_bic(FitSel sel, const int64_t* __restrict__ term_sample_off, const double* __restrict__ delays,
          const int32_t* __restrict__ counts, const double* __restrict__ mean_var,
          const double* __restrict__ cen_in, double* __restrict__ bic_out) {
  __shared__ double tab[64];
  __shared__ Fit fits[128 / 32];
  load_exp_table(tab);
  const int w = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  if (w >= sel.n_terms) return;
  double bic = INFINITY;
  int t;
  const double* draws;
  if (select_fit<K>(sel, counts, &t, &draws, nullptr)) {
    const int n = counts[t];
    double cen[KC];
#pragma unroll
    for (int j = 0; j < KC; ++j) cen[j] = j < K ? cen_in[(size_t)t * KC + j] : 0.0;
    Fit& f = fits[threadIdx.x >> 5];
    double sc = 0.0;
    if (em_fit<K, false>(delays + term_sample_off[t], n, mean_var[2 * t], cen, tab, f, true, &sc))
      bic = -2.0 * sc * (double)n + (double)(3 * K - 1) * log((double)n);   // GaussianMixture.bic, 'diag'
  }
  if ((threadIdx.x & 31) == 0) bic_out[(size_t)w * KC + (K - 1)] = bic;
}

// np.argmin over the BICs of the fits that did not raise (first minimum); terms without a fit get
// the degenerate record right here: services_times = (0, 0) -> sigma clamp (V3:765-766, V1:130-131).
// hist[k] counts the terms whose arg-min is k.
__global__ void k_gmm_select(int n_terms, const int32_t* __restrict__ max_n, const double* __restrict__ bic,
                             int32_t* __restrict__ best_k_out, uint32_t* __restrict__ hist,
                             double* __restrict__ mix_out, int32_t* __restrict__ n_selected_out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_terms) return;
  int best_k = 0;
  double best = INFINITY;
  for (int k = 1; k <= max_n[t]; ++k) {
    double b = bic[(size_t)t * KC + (k - 1)];
    if (b < best) { best = b; best_k = k; }
  }
  best_k_out[t] = best_k;
  if (best_k > 0) atomicAdd(&hist[best_k], 1u);
  else {
    double* rec = mix_out + (size_t)t * TW_MIX_REC;
    for (int q = 0; q < TW_MIX_REC; ++q) rec[q] = 0.0;
    rec[2] = 0.001;
    rec[3] = log(0.001);
    if (n_selected_out) n_selected_out[t] = 0;
  }
}

// terms grouped by their arg-min K: list[off_K + j], off_K = hist[1] + ... + hist[K-1]
__global__ void k_gmm_group(int n_terms, const int32_t* __restrict__ best_k, const uint32_t* __restrict__ hist,
                            uint32_t* __restrict__ cursor, int32_t* __restrict__ list) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_terms) return;
  const int k = best_k[t];
  if (k <= 0) return;
  uint32_t off = 0;
  for (int q = 1; q < k; ++q) off += hist[q];
  list[off + atomicAdd(&cursor[k], 1u)] = t;
}

// final 'full' fit of the terms whose BIC arg-min is K: dense warps over the grouped list
template <int K>
__global__ void __launch_bounds__(128, em_min_blocks(K))
k_gmm_final(FitSel sel, const int64_t* __restrict__ term_sample_off, const double* __restrict__ delays,
            const int32_t* __restrict__ counts, const double* __restrict__ mean_var,
            const double* __restrict__ cen_in, double* __restrict__ mix_out, int32_t* __restrict__ n_selected_out) {
  __shared__ double tab[64];
  __shared__ Fit fits[128 / 32];
  load_exp_table(tab);
  const unsigned w = (blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5;
  if (w >= sel.hist[K]) return;
  uint32_t off = 0;
#pragma unroll
  for (int q = 1; q < K; ++q) off += sel.hist[q];
  const int t = sel.list[off + w];
  const int lane = threadIdx.x & 31;
  const int n = counts[t];
  double cen[KC];
#pragma unroll
  for (int j = 0; j < KC; ++j) cen[j] = j < K ? cen_in[(size_t)t * KC + j] : 0.0;
  Fit& f = fits[threadIdx.x >> 5];
  const bool ok = em_fit<K, true>(delays + term_sample_off[t], n, mean_var[2 * t], cen, tab, f, false, nullptr);
  if (lane == 0) {
    double* rec = mix_out + (size_t)t * TW_MIX_REC;
    for (int q = 0; q < TW_MIX_REC; ++q) rec[q] = 0.0;
    if (ok) {
      rec[0] = (double)K;
#pragma unroll
      for (int c = 0; c < K; ++c) {
        rec[1 + c] = f.pc[c];
        rec[6 + c] = f.mu[c] * f.pc[c];
        rec[11 + c] = f.logpc[c];
        rec[16 + c] = f.logw[c];
      }
    } else {
      rec[2] = 0.001;
      rec[3] = log(0.001);
    }
    if (n_selected_out) n_selected_out[t] = ok ? K : 0;
  }
}

// ---- FP64 issue-rate micro-benchmark (the peak the refit's roofline is quoted against): every thread
// runs 8 independent DFMA chains; 2 flops per DFMA.
__global__ void __launch_bounds__(256)
k_fp64_peak(int iters, double* __restrict__ sink) {
  double a0 = threadIdx.x * 1e-9, a1 = a0 + 1e-3, a2 = a0 + 2e-3, a3 = a0 + 3e-3, a4 = a0 + 4e-3, a5 = a0 + 5e-3,
         a6 = a0 + 6e-3, a7 = a0 + 7e-3;
  const double m = 0.9999999, c = 1e-7;
  for (int i = 0; i < iters; ++i) {
    a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
    a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
  }
  const double r = ((a0 + a1) + (a2 + a3)) + ((a4 + a5) + (a6 + a7));
  if (r == 123.456) sink[0] = r;       // never true: keeps the chains alive
}

cudaError_t launch_fp64_peak(int blocks, int iters, double* sink, cudaStream_t s, int64_t& launches) {
  k_fp64_peak<<<blocks, 256, 0, s>>>(iters, sink);
  return after_launch(launches);
}

cudaError_t gmm_work_read(unsigned long long* out, bool reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out, g_gmm_em_evals, sizeof(unsigned long long));
  if (e != cudaSuccess) return e;
  if (reset) {
    const unsigned long long z = 0;
    e = cudaMemcpyToSymbol(g_gmm_em_evals, &z, sizeof z);
  }
  return e;
}

cudaError_t launch_gmm_prep(int n_terms, const int64_t* term_sample_off, const double* delays,
                            const int32_t* counts, int32_t* max_n, double* mean_var, cudaStream_t s,
                            int64_t& launches) {
  k_gmm_prep<<<(n_terms + 3) / 4, 128, 0, s>>>(n_terms, term_sample_off, delays, counts, max_n, mean_var);
  return after_launch(launches);
}

cudaError_t launch_gmm_skip(int n_problems, const int32_t* prob_ep_off, const int32_t* ep_term_off,
                            const int32_t* term_order, const int32_t* max_n, const uint32_t* prob_base_skip,
                            uint32_t* rng_skip, cudaStream_t s, int64_t& launches) {
  k_gmm_skip<<<(n_problems + 127) / 128, 128, 0, s>>>(n_problems, prob_ep_off, ep_term_off, term_order, max_n,
                                                       prob_base_skip, rng_skip);
  return after_launch(launches);
}

cudaError_t launch_gmm_draws(int n_problems, const int32_t* prob_ep_off, const int32_t* ep_term_off,
                             const int32_t* max_n, uint32_t* prob_draws, cudaStream_t s, int64_t& launches) {
  k_gmm_draws<<<(n_problems + 127) / 128, 128, 0, s>>>(n_problems, prob_ep_off, ep_term_off, max_n, prob_draws);
  return after_launch(launches);
}

template <int K>
static cudaError_t launch_fit_phases(const FitSel& sel, int n_warps, const int64_t* term_sample_off,
                                     const double* delays, const int32_t* counts, const double* mean_var,
                                     double* cen, int* err_flag, cudaStream_t s, int64_t& launches) {
  const int blocks = (n_warps + 3) / 4;
  k_gmm_seed<K><<<blocks, 128, 0, s>>>(sel, term_sample_off, delays, counts, mean_var, cen, err_flag);
  cudaError_t e = after_launch(launches);
  if (e != cudaSuccess) return e;
  k_gmm_lloyd<K><<<blocks, 128, 0, s>>>(sel, term_sample_off, delays, counts, mean_var, cen);
  return after_launch(launches);
}

// fork: every side stream waits for the work queued on s so far; join: s waits for every side stream
static cudaError_t fork_streams(GmmFork* fk, cudaStream_t s) {
  cudaError_t e = cudaEventRecord(fk->fork, s);
  for (int q = 0; q < TW_GMM_MAX_COMP && e == cudaSuccess; ++q) e = cudaStreamWaitEvent(fk->side[q], fk->fork, 0);
  return e;
}
static cudaError_t join_streams(GmmFork* fk, cudaStream_t s) {
  cudaError_t e = cudaSuccess;
  for (int q = 0; q < TW_GMM_MAX_COMP && e == cudaSuccess; ++q) {
    e = cudaEventRecord(fk->join[q], fk->side[q]);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(s, fk->join[q], 0);
  }
  return e;
}

// `cen` holds one [n_terms x 5] slab per component count: the five fit chains (seed -> Lloyd -> EM
// for K = 5..1) only share read-only inputs, so each runs on its own side stream; kernels of
// different chains then overlap (the EM kernels are FP64-issue bound, the k-means kernels latency
// bound) and the chains' tails hide behind each other.
cudaError_t launch_gmm_fit(int n_terms, const int64_t* term_sample_off, const double* delays,
                           const int32_t* counts, const int32_t* max_n, const double* mean_var,
                           const uint32_t* rng_skip, const double* stream, int stream_len,
                           const double* stream100, double* bic, double* cen, double* mix_out,
                           int32_t* n_selected_out, int* err_flag, GmmFork* fk, cudaStream_t s,
                           int64_t& launches) {
  cudaError_t e;
  const int blocks = (n_terms + 3) / 4;
  const size_t slab = (size_t)n_terms * KC;
  const FitSel sel{nullptr, nullptr, max_n, rng_skip, stream, stream_len, n_terms};
  e = fork_streams(fk, s);
  if (e != cudaSuccess) return e;
#define TW_BIC(K)                                                                                          \
  {                                                                                                        \
    cudaStream_t q = fk->side[K - 1];                                                                      \
    double* c = cen + (K - 1) * slab;                                                                      \
    e = launch_fit_phases<K>(sel, n_terms, term_sample_off, delays, counts, mean_var, c, err_flag, q,      \
                             launches);                                                                    \
    if (e != cudaSuccess) return e;                                                                        \
    k_gmm_bic<K><<<blocks, 128, 0, q>>>(sel, term_sample_off, delays, counts, mean_var, c, bic);           \
    e = after_launch(launches);                                                                            \
    if (e != cudaSuccess) return e;                                                                        \
  }
  TW_BIC(5) TW_BIC(4) TW_BIC(3) TW_BIC(2) TW_BIC(1)     // longest fits first
#undef TW_BIC
  e = join_streams(fk, s);
  if (e != cudaSuccess) return e;
  // group the terms by selected K so that the final fits run with every warp busy.  Scratch:
  // rng_skip (free after the BIC fits) -> hist[0..7], cursor[8..15]; bic (free after the select
  // kernel) -> the grouped list; max_n -> best_k.
  uint32_t* hist = const_cast<uint32_t*>(rng_skip);
  uint32_t* cursor = hist + 8;
  int32_t* best_k = const_cast<int32_t*>(max_n);
  int32_t* list = reinterpret_cast<int32_t*>(bic);
  e = cudaMemsetAsync(hist, 0, 16 * sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  k_gmm_select<<<(n_terms + 127) / 128, 128, 0, s>>>(n_terms, max_n, bic, best_k, hist, mix_out, n_selected_out);
  e = after_launch(launches);
  if (e != cudaSuccess) return e;
  k_gmm_group<<<(n_terms + 127) / 128, 128, 0, s>>>(n_terms, best_k, hist, cursor, list);
  e = after_launch(launches);
  if (e != cudaSuccess) return e;
  const FitSel fin{list, hist, nullptr, nullptr, stream100, 16, n_terms};
  e = fork_streams(fk, s);
  if (e != cudaSuccess) return e;
#define TW_FINAL(K)                                                                                        \
  {                                                                                                        \
    cudaStream_t q = fk->side[K - 1];                                                                      \
    double* c = cen + (K - 1) * slab;                                                                      \
    e = launch_fit_phases<K>(fin, n_terms, term_sample_off, delays, counts, mean_var, c, nullptr, q,       \
                             launches);                                                                    \
    if (e != cudaSuccess) return e;                                                                        \
    k_gmm_final<K><<<blocks, 128, 0, q>>>(fin, term_sample_off, delays, counts, mean_var, c, mix_out,      \
                                          n_selected_out);                                                 \
    e = after_launch(launches);                                                                            \
    if (e != cudaSuccess) return e;                                                                        \
  }
  TW_FINAL(5) TW_FINAL(4) TW_FINAL(3) TW_FINAL(2) TW_FINAL(1)
#undef TW_FINAL
  return join_streams(fk, s);
}

}  // namespace tw
