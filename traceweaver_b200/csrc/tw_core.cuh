// tw_core.cuh — per-thread building blocks of the span-assignment engine.
//
// Everything here is `__host__ __device__` on purpose: the CUDA kernels (tw_score.cu,
// tw_stitch.cu, ...) are thin cooperative wrappers around these functions, and the build
// container has no GPU, so tests/emul/ compiles the SAME functions with g++ and steps the kernels'
// thread loops sequentially to unit-test the device logic on CPU.  That harness is test
// infrastructure; the shipped library contains only the CUDA path.
//
// Reference semantics (file:line are in /root/reference/src/trace_reconstructor/ports/python/
// algorithms/): V3 = traceweaver_v3.py, V1 = traceweaver_v1.py.
#pragma once
#include <stdint.h>
#include <string.h>
#include <math.h>

#include "../../include/traceweaver_b200.h"

#if defined(__CUDACC__)
#define TW_HD __host__ __device__ __forceinline__
#define TW_HD_NOINLINE __host__ __device__
#else
#define TW_HD inline
#define TW_HD_NOINLINE
#endif

#define TW_MAX_TERMS 48  // <= E(E-1)/2 primary edges + E roots + E lasts for E = 8
#define TW_LOG_SQRT_2PI 0.91893853320467274178032973640562
#define TW_LOG_2PI 1.8378770664093453

namespace tw {

// IEEE-exact f64 ops that the compiler may not contract into FMAs: scores must follow
// scipy/sklearn operation order (contract: |delta| <= 1e-5, in practice ~1e-13).
#if defined(__CUDA_ARCH__)
TW_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
TW_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
TW_HD double dsub(double a, double b) { return __dsub_rn(a, b); }
TW_HD double ddiv(double a, double b) { return __ddiv_rn(a, b); }
#else
TW_HD double dmul(double a, double b) { volatile double r = a * b; return r; }
TW_HD double dadd(double a, double b) { volatile double r = a + b; return r; }
TW_HD double dsub(double a, double b) { volatile double r = a - b; return r; }
TW_HD double ddiv(double a, double b) { volatile double r = a / b; return r; }
#endif

// ---------------------------------------------------------------------------------------------
// Likelihood terms: GetEpPairCost, V1:117-139.
// ---------------------------------------------------------------------------------------------

// scipy.stats.norm.logpdf(dt, mu, sigma) = -x^2/2 - log(sqrt(2 pi)) - log(sigma); rec = {mu,
// sigma (already clamped, V1:130-131), log(sigma)}.
TW_HD double gauss_logpdf(const double* rec, double dt) {
  double x = ddiv(dsub(dt, rec[0]), rec[1]);
  return dsub(dsub(-dmul(x, x) / 2.0, TW_LOG_SQRT_2PI), rec[2]);
}

// sklearn GaussianMixture.score of one sample (V1:125-126): logsumexp_k(log N_k + log w_k).
// rec = {k, pc[5], mu*pc[5], log pc[5], log w[5]}; k == 0: Gaussian record at rec+1.
TW_HD double mix_logpdf(const double* rec, double dt) {
  int k = (int)rec[0];
  if (k == 0) return gauss_logpdf(rec + 1, dt);
  double a[TW_GMM_MAX_COMP];
  double amax = -INFINITY;
#pragma unroll
  for (int c = 0; c < TW_GMM_MAX_COMP; ++c) {
    if (c < k) {
      double y = dsub(dmul(dt, rec[1 + c]), rec[6 + c]);
      a[c] = dadd(dadd(dmul(-0.5, dadd(TW_LOG_2PI, dmul(y, y))), rec[11 + c]), rec[16 + c]);
      if (a[c] > amax) amax = a[c];
    }
  }
  double s = 0.0, m = 0.0;
#pragma unroll
  for (int c = 0; c < TW_GMM_MAX_COMP; ++c) {
    if (c < k) {
      if (a[c] == amax) m += 1.0;
      else s = dadd(s, exp(dsub(a[c], amax)));
    }
  }
  if (m > 1.0) return dadd(dadd(log1p(ddiv(s, m)), log(m)), amax);
  return dadd(log1p(s), amax);   // log(1) == 0 exactly
}

// ---------------------------------------------------------------------------------------------
// Problem view (one service).  Pointers are problem-local bases into the batch arrays.
// ---------------------------------------------------------------------------------------------
struct ProbView {
  int E, n_in, n_terms;
  int ep0, term0;
  int64_t in_off, tuple_off;
  const int64_t* is;
  const int64_t* ie;
  const int64_t* os[TW_MAX_E];
  const int64_t* oe[TW_MAX_E];
  int64_t out_off[TW_MAX_E];
  int n_out[TW_MAX_E];
  uint32_t pred[TW_MAX_E];
  int term_lo[TW_MAX_E + 1];
  int8_t term_src[TW_MAX_TERMS];
};

TW_HD_NOINLINE inline int load_view(const tw_batch& b, int p, ProbView& v) {
  v.ep0 = b.prob_ep_off[p];
  v.E = b.prob_ep_off[p + 1] - v.ep0;
  if (v.E < 1 || v.E > TW_MAX_E) return TW_ERR_INVALID;
  v.in_off = b.prob_in_off[p];
  v.n_in = (int)(b.prob_in_off[p + 1] - v.in_off);
  v.tuple_off = b.prob_tuple_off[p];
  v.is = b.in_start + v.in_off;
  v.ie = b.in_end + v.in_off;
  v.term0 = b.ep_term_off[v.ep0];
  v.n_terms = b.ep_term_off[v.ep0 + v.E] - v.term0;
  if (v.n_terms > TW_MAX_TERMS) return TW_ERR_INVALID;
  for (int e = 0; e < v.E; ++e) {
    int64_t o = b.ep_out_off[v.ep0 + e];
    v.out_off[e] = o;
    v.os[e] = b.out_start + o;
    v.oe[e] = b.out_end + o;
    v.n_out[e] = (int)(b.ep_out_off[v.ep0 + e + 1] - o);
    v.pred[e] = b.ep_pred_mask[v.ep0 + e];
    v.term_lo[e] = b.ep_term_off[v.ep0 + e] - v.term0;
  }
  v.term_lo[v.E] = v.n_terms;
  for (int t = 0; t < v.n_terms; ++t) v.term_src[t] = b.term_src[v.term0 + t];
  return TW_OK;
}

// Parameters as seen by one in-span: `gauss` points at the [n_terms][3] table of its 100-span
// batch (V3:1173-1178), `mix` at the problem's [n_terms][21] table.
struct ParamView {
  int mode;
  const double* gauss;
  const double* mix;
  const double* etab = nullptr;   // device: shared-memory copy of c_exp2_64 -> branch-free mixture path
};

#ifdef __CUDACC__
// exp(d) for d in [-40, 0], branch free (callers discard the value for d < -40): d = (64 q + j) ln2/64
// + r, |r| <= ln2/128, exp(d) = 2^q * 2^(j/64) * P5(r).  ~1.5 ulp; ten FP64 operations and no slow
// path, so independent evaluations interleave instead of serialising behind libdevice's range
// branches.  `tab` is a shared-memory copy of c_exp2_64 (a divergent index would serialise in the
// constant cache).
static __constant__ double c_exp2_64[64] = {
    1.0, 1.0108892860517005, 1.0218971486541166, 1.0330248790212284,
    1.0442737824274138, 1.0556451783605572, 1.0671404006768237, 1.0787607977571199,
    1.0905077326652577, 1.102382583307841, 1.1143867425958924, 1.1265216186082418,
    1.1387886347566916, 1.1511892299529827, 1.1637248587775775, 1.1763969916502812,
    1.189207115002721, 1.202156731452703, 1.215247359980469, 1.22848053610687,
    1.241857812073484, 1.255380757024691, 1.2690509571917332, 1.2828700160787783,
    1.2968395546510096, 1.3109612115247644, 1.3252366431597413, 1.339667524053303,
    1.3542555469368927, 1.3690024229745905, 1.383909881963832, 1.3989796725383112,
    1.4142135623730951, 1.42961333839197, 1.4451808069770467, 1.460917794180647,
    1.4768261459394993, 1.4929077282912648, 1.5091644275934228, 1.5255981507445384,
    1.5422108254079407, 1.559004400237837, 1.5759808451078865, 1.593142151342267,
    1.6104903319492543, 1.6280274218573478, 1.645755478153965, 1.6636765803267364,
    1.681792830507429, 1.7001063537185235, 1.718619298122478, 1.7373338352737062,
    1.7562521603732995, 1.7753764925265212, 1.7947090750031072, 1.8142521755003989,
    1.8340080864093424, 1.8539791250833855, 1.8741676341103, 1.8945759815869656,
    1.9152065613971474, 1.9360617934922943, 1.9571441241754002, 1.978456026387951};

__device__ __forceinline__ void load_exp_table(double* tab) {   // block-wide; call before any early return
  for (int x = threadIdx.x; x < 64; x += blockDim.x) tab[x] = c_exp2_64[x];
  __syncthreads();
}

__device__ __forceinline__ double exp_neg(const double* __restrict__ tab, double d) {
  const double kMagic = 6755399441055744.0;                     // 1.5 * 2^52: rint() in the low word
  const double t = fma(d, 92.33248261689366, kMagic);           // 64 / ln 2
  const int n = __double2loint(t);
  const double nf = t - kMagic;
  double r = fma(nf, -0.010830424667801708, d);                 // ln2/64, high 29 bits: n * hi is exact
  r = fma(nf, -2.8447437476627285e-11, r);
  double p = 1.0 / 120.0;
  p = fma(p, r, 1.0 / 24.0);
  p = fma(p, r, 1.0 / 6.0);
  p = fma(p, r, 0.5);
  p = fma(p, r, 1.0);
  p = fma(p, r, 1.0);
  const double v = tab[n & 63] * p;
  return __hiloint2double(__double2hiint(v) + ((n >> 6) << 20), __double2loint(v));
}

// mix_logpdf with every component evaluated unconditionally (records are zero beyond k) and masked,
// the exponentials from exp_neg: logsumexp = max + log(sum exp(a_c - max)), the maximum's term
// being exactly 1.  Same per-component operation order as mix_logpdf; the result differs from it
// by the rounding of exp / log only (~1e-16 relative).
__device__ __forceinline__ double mix_logpdf_tab(const double* rec, double dt, const double* __restrict__ tab) {
  const int k = (int)rec[0];
  if (k == 0) return gauss_logpdf(rec + 1, dt);
  double a[TW_GMM_MAX_COMP];
  double amax = -INFINITY;
#pragma unroll
  for (int c = 0; c < TW_GMM_MAX_COMP; ++c) {
    const double y = dsub(dmul(dt, rec[1 + c]), rec[6 + c]);
    const double w = dadd(dadd(dmul(-0.5, dadd(TW_LOG_2PI, dmul(y, y))), rec[11 + c]), rec[16 + c]);
    a[c] = c < k ? w : -INFINITY;
    amax = a[c] > amax ? a[c] : amax;
  }
  double s = 0.0;
#pragma unroll
  for (int c = 0; c < TW_GMM_MAX_COMP; ++c) {
    const double d = a[c] - amax;
    const double e = exp_neg(tab, d);
    s += d >= -40.0 ? e : 0.0;      // exp(d) < 2^-57 cannot change a sum that holds the maximum's 1.0
  }
  return dadd(log(s), amax);
}
// mix_logpdf_tab for callers whose whole warp evaluates the SAME record (k is warp-uniform): only the
// k live components are computed.  Component for component the same operations in the same order as
// mix_logpdf_tab (whose masked components add an exact 0.0), so the value is bit-identical.
__device__ __forceinline__ double mix_logpdf_tab_uniform(const double* rec, double dt, const double* __restrict__ tab) {
  const int k = (int)rec[0];
  if (k == 0) return gauss_logpdf(rec + 1, dt);
  double a[TW_GMM_MAX_COMP];
  double amax = -INFINITY;
#pragma unroll
  for (int c = 0; c < TW_GMM_MAX_COMP; ++c) {
    if (c < k) {
      const double y = dsub(dmul(dt, rec[1 + c]), rec[6 + c]);
      a[c] = dadd(dadd(dmul(-0.5, dadd(TW_LOG_2PI, dmul(y, y))), rec[11 + c]), rec[16 + c]);
      amax = a[c] > amax ? a[c] : amax;
    }
  }
  double s = 0.0;
#pragma unroll
  for (int c = 0; c < TW_GMM_MAX_COMP; ++c) {
    if (c < k) {
      const double d = a[c] - amax;
      const double e = exp_neg(tab, d);
      s += d >= -40.0 ? e : 0.0;
    }
  }
  return dadd(log(s), amax);
}
#endif

TW_HD double term_logpdf(const ParamView& pv, int t, double dt) {
  if (pv.mode == TW_PARAMS_GAUSS_BATCHED) return gauss_logpdf(pv.gauss + t * TW_GAUSS_REC, dt);
#ifdef __CUDA_ARCH__
  if (pv.etab) return mix_logpdf_tab(pv.mix + t * TW_MIX_REC, dt, pv.etab);
#endif
  return mix_logpdf(pv.mix + t * TW_MIX_REC, dt);
}

// A window of an ep's out list: element x of the window is original index base + x.  The score
// kernel points these at shared-memory staged copies, the stitch kernel at the global arrays.
struct OutWin {
  const int64_t* s;
  const int64_t* e;
  int base;
  int n;
};

// ScoreAssignmentAsPerInvocationGraph, V1:305-361 (no skips, normalized = False).
// cs/ce = start/end of the chosen out span per ep.
TW_HD double score_tuple(const ProbView& v, const ParamView& pv, int64_t in_s, int64_t in_e,
                         const int64_t* cs, const int64_t* ce) {
  int last = 0;  // max(..., key = end) keeps the first maximum (V1:314)
  for (int e = 1; e < v.E; ++e)
    if (ce[e] > ce[last]) last = e;
  double cost = 0.0;
  for (int e = 0; e < v.E; ++e) {
    for (int t = v.term_lo[e]; t < v.term_lo[e + 1]; ++t) {
      int src = v.term_src[t];
      int64_t d;
      if (src >= 0) d = cs[e] - ce[src];                  // V1:345
      else if (src == TW_TERM_ROOT) d = cs[e] - in_s;     // V1:349-350
      else {                                              // V1:354-355
        if (e != last) continue;
        d = in_e - ce[e];
      }
      cost = dadd(cost, term_logpdf(pv, t, (double)d));
    }
  }
  return cost;
}

// ---------------------------------------------------------------------------------------------
// A GIVEN tuple of in-span i (tw_score_assignments): feasibility code, score, margin.
// `assign` is the batch's tw_pass_out.assign array; tks / tki (NULL: no margin) are the in-span's
// row of a final top-K list (score[K], idx[K][E]) holding tk_cnt entries.
// ---------------------------------------------------------------------------------------------
struct Assessment {
  double score;
  double margin;
  int code;
};

TW_HD Assessment assess_in_span(const ProbView& v, const ParamView& pv, int i, const int32_t* assign,
                                const double* tks, const int32_t* tki, int tk_cnt) {
  Assessment a{NAN, NAN, TW_ASSESS_SCORED};
  int c[TW_MAX_E];
  bool na = false, range = false;
  for (int e = 0; e < v.E; ++e) {
    c[e] = assign[v.tuple_off + (int64_t)e * v.n_in + i];
    if (c[e] == -1) na = true;
    else if (c[e] < 0 || c[e] >= v.n_out[e]) range = true;
  }
  if (na || range) {
    a.code = na ? TW_ASSESS_NA : TW_ASSESS_RANGE;
    return a;
  }
  const int64_t in_s = v.is[i], in_e = v.ie[i];
  int64_t cs[TW_MAX_E] = {}, ce[TW_MAX_E] = {};
  bool inside = true;
  for (int e = 0; e < v.E; ++e) {
    cs[e] = v.os[e][c[e]];
    ce[e] = v.oe[e][c[e]];
    if (cs[e] < in_s || ce[e] > in_e) inside = false;              // V3:328-333
  }
  if (!inside) {
    a.code = TW_ASSESS_CONTAIN;
    return a;
  }
  for (int e = 0; e < v.E; ++e)                                      // V3:335-347: every DAG edge
    for (int b = 0; b < e; ++b)
      if ((v.pred[e] >> b & 1u) && ce[b] > cs[e]) {
        a.code = TW_ASSESS_ORDER;
        return a;
      }
  a.score = score_tuple(v, pv, in_s, in_e, cs, ce);
  if (tks && tk_cnt > 0) {
    bool top = true;
    for (int e = 0; e < v.E; ++e) top = top && tki[e] == c[e];
    a.margin = !top ? dsub(a.score, tks[0]) : tk_cnt > 1 ? dsub(tks[0], tks[1]) : INFINITY;
  }
  return a;
}

// ---------------------------------------------------------------------------------------------
// Top-K list: V3:305-307 keeps the K largest (score, stack); V3:461 sorts descending.  Order:
// score, then the first tuple position whose span differs decides by start (spans.py:51).
// ---------------------------------------------------------------------------------------------
struct TopK {
  double score[TW_K + 1];
  int idx[TW_K + 1][TW_MAX_E];
  uint8_t heap[TW_K + 1];   // heap[0..n) = slots in CPython heapq array order; heap[n] = a free slot
  int n;
  TW_HD void clear() {
    n = 0;
    for (int k = 0; k <= TW_K; ++k) heap[k] = (uint8_t)k;
  }
};

// a < b in the reference's (score, stack) order: tuple comparison takes the score first; on equal
// scores the stacks are compared element by element, the first position holding two different Span
// objects decides by Span.__lt__ = start_mus (spans.py:51).  Two different spans with the same start
// are neither smaller: a < b and b < a are both false, and then the ORDER OF THE OPERATIONS decides
// where the entries end up — which is why topk_offer below replays heapq itself.
TW_HD bool cand_less(const ProbView& v, double sa, const int* ca, double sb, const int* cb) {
  if (sa < sb) return true;
  if (!(sa == sb)) return false;
  for (int e = 0; e < v.E; ++e)
    if (ca[e] != cb[e]) {
      // skip spans (negative codes, tw_skip.cu) have no start time: the reference raises when it compares
      // one with a real span; the skip kernel reports that case before it gets here
      if (ca[e] < 0 || cb[e] < 0) return false;
      return v.os[e][ca[e]] < v.os[e][cb[e]];
    }
  return false;
}

TW_HD bool topk_slot_less(const ProbView& v, const TopK& tk, int a, int b) {
  return cand_less(v, tk.score[a], tk.idx[a], tk.score[b], tk.idx[b]);
}

// heapq._siftdown: the entry at `pos` moves towards the root while it is smaller than its parent
TW_HD void topk_toward_root(const ProbView& v, TopK& tk, int startpos, int pos) {
  const uint8_t item = tk.heap[pos];
  while (pos > startpos) {
    const int parent = (pos - 1) >> 1;
    if (!topk_slot_less(v, tk, item, tk.heap[parent])) break;
    tk.heap[pos] = tk.heap[parent];
    pos = parent;
  }
  tk.heap[pos] = item;
}

// heapq._siftup: the smaller child is pulled up all the way to a leaf (the right child on
// "not left < right"), the displaced entry is placed there and moved back towards the root
TW_HD void topk_toward_leaf(const ProbView& v, TopK& tk, int pos) {
  const int startpos = pos, endpos = tk.n;
  const uint8_t item = tk.heap[pos];
  int child = 2 * pos + 1;
  while (child < endpos) {
    const int right = child + 1;
    if (right < endpos && !topk_slot_less(v, tk, tk.heap[child], tk.heap[right])) child = right;
    tk.heap[pos] = tk.heap[child];
    pos = child;
    child = 2 * pos + 1;
  }
  tk.heap[pos] = item;
  topk_toward_root(v, tk, startpos, pos);
}

// V3:305-307: heapq.heappush(top_assignments, (score, stack)); if len > K: heapq.heappop(...).
// Replayed literally (min-heap of at most K + 1 entries in heapq's array layout), so that the
// surviving entries AND their array order are the reference's also when entries compare equal.
TW_HD void topk_offer(const ProbView& v, TopK& tk, double score, const int* c) {
  // A full heap and a score strictly below the root's: heappush moves the new entry to the root
  // (its score is below every entry's) and heappop takes it out again, the last entry returning to
  // the place it left — the array is exactly what it was.  Nothing to do (the common case once K good
  // tuples are in).
  if (tk.n == TW_K && score < tk.score[tk.heap[0]]) return;
  const int slot = tk.heap[tk.n];
  tk.score[slot] = score;
  for (int e = 0; e < v.E; ++e) tk.idx[slot][e] = c[e];
  tk.n += 1;
  topk_toward_root(v, tk, 0, tk.n - 1);
  if (tk.n > TW_K) {                     // heappop: the last entry replaces the root
    const uint8_t last = tk.heap[tk.n - 1], root = tk.heap[0];
    tk.n -= 1;
    tk.heap[tk.n] = root;                // the popped entry's slot is the free one
    if (tk.n > 0) {
      tk.heap[0] = last;
      topk_toward_leaf(v, tk, 0);
    }
  }
}

// V3:461 `top_assignments.sort(reverse=True)`: a stable descending sort of the heap ARRAY (entries
// that compare equal keep their array order).  Leaves rank k in score[k] / idx[k].
TW_HD void topk_finish(const ProbView& v, TopK& tk) {
  uint8_t ord[TW_K + 1];
  for (int a = 0; a < tk.n; ++a) {
    const uint8_t x = tk.heap[a];
    int j = a - 1;
    while (j >= 0 && topk_slot_less(v, tk, ord[j], x)) { ord[j + 1] = ord[j]; --j; }
    ord[j + 1] = x;
  }
  double sc[TW_K];
  int ix[TW_K][TW_MAX_E];
  for (int k = 0; k < tk.n; ++k) {
    sc[k] = tk.score[ord[k]];
    for (int e = 0; e < v.E; ++e) ix[k][e] = tk.idx[ord[k]][e];
  }
  for (int k = 0; k < tk.n; ++k) {
    tk.score[k] = sc[k];
    for (int e = 0; e < v.E; ++e) tk.idx[k][e] = ix[k][e];
  }
}

// Sorted-list variant (insert keeping the list descending; an entry that compares equal to a listed
// one goes behind it).  Only exact where no two tuples compare equal; used to merge partial lists.
TW_HD void topk_offer_sorted(const ProbView& v, TopK& tk, double score, const int* c) {
  int pos = tk.n;
  while (pos > 0 && cand_less(v, tk.score[pos - 1], tk.idx[pos - 1], score, c)) --pos;
  if (pos >= TW_K) return;
  int last = tk.n < TW_K ? tk.n : TW_K - 1;
  for (int k = last; k > pos; --k) {
    tk.score[k] = tk.score[k - 1];
    for (int e = 0; e < v.E; ++e) tk.idx[k][e] = tk.idx[k - 1][e];
  }
  tk.score[pos] = score;
  for (int e = 0; e < v.E; ++e) tk.idx[pos][e] = c[e];
  if (tk.n < TW_K) tk.n++;
}

// ---------------------------------------------------------------------------------------------
// Candidate enumeration: DfsTraverseX V3:292-351 / DfsTraverse3 V3:236-288 in the no-skip
// regime.  Feasible tuples = one not-taken out span per ep with
//     in.start <= s.start, s.end <= in.end                      (V3:328-333)
//     c_b.end <= s.start for every DAG predecessor b of the ep   (V3:335-347)
// FindCutoffs (V3:182-217) only narrows the scan and never removes a feasible tuple (a feasible
// c_e has c_e.start <= c_e.end <= c_s.start for every successor s), so it is not reproduced; the
// scan per ep is [lo_e, first span with start > in.end).  The oracle keeps the literal cutoffs,
// and parity between the two is what tests assert.
//
// Leaf is called with the original indices c[e] and the chosen spans' start/end.
// Taken is `bool(int ep, int orig_index)`.
// ---------------------------------------------------------------------------------------------
template <class Taken, class Leaf>
TW_HD void enumerate(const ProbView& v, int64_t in_s, int64_t in_e, const OutWin* w, const int* lo,
                     Taken taken, Leaf leaf) {
  int x[TW_MAX_E];
  int c[TW_MAX_E];
  int64_t cs[TW_MAX_E], ce[TW_MAX_E];
  int e = 0;
  x[0] = lo[0];
  while (e >= 0) {
    bool descended = false;
    while (x[e] < w[e].n) {
      int xi = x[e]++;
      int64_t s = w[e].s[xi];
      if (s > in_e) { x[e] = w[e].n; break; }   // sorted by start: nothing further fits
      int64_t en = w[e].e[xi];
      if (en > in_e) continue;
      uint32_t pm = v.pred[e];
      bool ok = true;
      for (int b = 0; b < e; ++b)
        if ((pm >> b & 1u) && ce[b] > s) { ok = false; break; }
      if (!ok) continue;
      int orig = w[e].base + xi;
      if (taken(e, orig)) continue;
      c[e] = orig; cs[e] = s; ce[e] = en;
      if (e == v.E - 1) { leaf(c, cs, ce); continue; }
      ++e;
      x[e] = lo[e];
      descended = true;
      break;
    }
    if (!descended) --e;
  }
}

// ---------------------------------------------------------------------------------------------
// Term tables.  The score of a tuple is a sum of terms that each depend on ONE candidate (root,
// last) or on a PAIR of candidates (primary edge), so all distinct term values of an in-span fit
// a small table: for ep e with r_e candidates in range, r_e values per root/last term and
// r_b * r_e per edge term b->e.  The kernels (1) lay the tables of a tile / window out
// back to back in shared memory, (2) write (term id, dt) into every slot, (3) evaluate all slots
// with every lane busy — this is where the FP64 exp/log/div work of GetEpPairCost (V1:117-139)
// goes — and (4) run the DFS with look-ups only.  Values and summation order are unchanged, so
// scores are bit-identical to evaluating each leaf from scratch.
//
// Slot id byte: bits 0-5 = problem-local term index (< TW_MAX_TERMS), bits 6-7 = parameter batch
// relative to the tile's / window's first batch (pass 0 has one Gaussian table per 100 in-spans);
// 0xFF = slot no feasible tuple can use (candidate outside the in-span, taken, or pair out of order).
// ---------------------------------------------------------------------------------------------
#define TW_SLOT_INVALID 0xFF

// spans of the window from `lo` on whose start is <= in_e (the in-span's candidate range of one ep)
TW_HD int range_len(const OutWin& w, int lo, int64_t in_e) {
  int x = lo;
  while (x < w.n && w.s[x] <= in_e) ++x;
  return x - lo;
}

TW_HD int term_table_size(const ProbView& v, const int* r) {
  int tot = 0;
  for (int e = 0; e < v.E; ++e)
    for (int t = v.term_lo[e]; t < v.term_lo[e + 1]; ++t) {
      int src = v.term_src[t];
      tot += src >= 0 ? r[src] * r[e] : r[e];
    }
  return tot;
}

// offset of the LAST term's sub-table of every ep (its slot ids double as candidate validity)
TW_HD void term_table_last_offsets(const ProbView& v, const int* r, int* o_last) {
  int o = 0;
  for (int e = 0; e < v.E; ++e)
    for (int t = v.term_lo[e]; t < v.term_lo[e + 1]; ++t) {
      int src = v.term_src[t];
      if (src == TW_TERM_LAST) o_last[e] = o;
      o += src >= 0 ? r[src] * r[e] : r[e];
    }
}

// Writes dt (as double) and the slot id of every entry.  `brel` = parameter batch of this in-span
// relative to the tile / window base.  Taken is `bool(int ep, int orig_index)`.
template <class Taken>
TW_HD void term_table_fill(const ProbView& v, int64_t in_s, int64_t in_e, const OutWin* w, const int* lo,
                           const int* r, const int* o_last, int brel, Taken taken, double* tbl,
                           uint8_t* sid) {
  const uint8_t bb = (uint8_t)(brel << 6);
  // candidate validity first (LAST sub-tables): contained and not taken (V3:328-333)
  for (int e = 0; e < v.E; ++e) {
    const int t_last = v.term_lo[e + 1] - 1;
    for (int x = 0; x < r[e]; ++x) {
      int64_t en = w[e].e[lo[e] + x];
      bool ok = en <= in_e && !taken(e, w[e].base + lo[e] + x);
      tbl[o_last[e] + x] = (double)(in_e - en);                                    // V1:354-355
      sid[o_last[e] + x] = ok ? (uint8_t)(t_last | bb) : (uint8_t)TW_SLOT_INVALID;
    }
  }
  int o = 0;
  for (int e = 0; e < v.E; ++e)
    for (int t = v.term_lo[e]; t < v.term_lo[e + 1]; ++t) {
      int src = v.term_src[t];
      if (src >= 0) {                                                              // V1:345
        for (int xb = 0; xb < r[src]; ++xb) {
          bool vb = sid[o_last[src] + xb] != TW_SLOT_INVALID;
          int64_t eb = w[src].e[lo[src] + xb];
          for (int xe = 0; xe < r[e]; ++xe) {
            int64_t s = w[e].s[lo[e] + xe];
            bool ok = vb && eb <= s && sid[o_last[e] + xe] != TW_SLOT_INVALID;
            tbl[o] = (double)(s - eb);
            sid[o] = ok ? (uint8_t)(t | bb) : (uint8_t)TW_SLOT_INVALID;
            ++o;
          }
        }
      } else if (src == TW_TERM_ROOT) {                                            // V1:349-350
        for (int xe = 0; xe < r[e]; ++xe) {
          tbl[o] = (double)(w[e].s[lo[e] + xe] - in_s);
          sid[o] = sid[o_last[e] + xe] != TW_SLOT_INVALID ? (uint8_t)(t | bb) : (uint8_t)TW_SLOT_INVALID;
          ++o;
        }
      } else {
        o += r[e];
      }
    }
}

// score of a tuple from evaluated tables: same terms, same order as score_tuple()
TW_HD double table_score(const ProbView& v, const int* r, const int* lo_abs, const double* tbl, const int* c,
                         const int64_t* ce) {
  int last = 0;
  for (int e = 1; e < v.E; ++e)
    if (ce[e] > ce[last]) last = e;
  double cost = 0.0;
  int o = 0;
  for (int e = 0; e < v.E; ++e) {
    const int xe = c[e] - lo_abs[e];
    for (int t = v.term_lo[e]; t < v.term_lo[e + 1]; ++t) {
      int src = v.term_src[t];
      if (src >= 0) {
        cost = dadd(cost, tbl[o + (c[src] - lo_abs[src]) * r[e] + xe]);
        o += r[src] * r[e];
      } else {
        if (src == TW_TERM_ROOT || e == last) cost = dadd(cost, tbl[o + xe]);
        o += r[e];
      }
    }
  }
  return cost;
}

// ---------------------------------------------------------------------------------------------
// Lane-parallel form of the enumeration for in-spans with many candidate tuples.  The candidate
// product space prod_e r_e is indexed x0-major ("combo"), so ascending combo order IS the DFS leaf
// order of enumerate().  Lanes take combos first, first+step, ...; a combo is a feasible tuple iff
// every candidate slot is valid (term_table_fill) and every DAG edge is ordered (V3:335-347).
// Leaf(c, ce, combo).
// ---------------------------------------------------------------------------------------------
TW_HD long long combo_count(const ProbView& v, const int* r) {
  long long p = 1;
  for (int e = 0; e < v.E; ++e) {
    p *= r[e];
    if (p > (1LL << 40)) return 1LL << 40;
  }
  return p;
}

template <class Leaf>
TW_HD void enumerate_combos(const ProbView& v, const OutWin* w, const int* lo, const int* r, const int* o_last,
                            const uint8_t* sid, long long first, long long step, long long P, Leaf leaf) {
  for (long long combo = first; combo < P; combo += step) {
    int x[TW_MAX_E], c[TW_MAX_E];
    int64_t cs[TW_MAX_E], ce[TW_MAX_E];
    long long idx = combo;
    bool ok = true;
    for (int e = v.E - 1; e >= 0; --e) {
      x[e] = (int)(idx % r[e]);
      idx /= r[e];
      if (sid[o_last[e] + x[e]] == TW_SLOT_INVALID) ok = false;
    }
    if (!ok) continue;
    for (int e = 0; e < v.E && ok; ++e) {
      cs[e] = w[e].s[lo[e] + x[e]];
      ce[e] = w[e].e[lo[e] + x[e]];
      c[e] = w[e].base + lo[e] + x[e];
      uint32_t pm = v.pred[e];
      for (int b = 0; b < e; ++b)
        if ((pm >> b & 1u) && ce[b] > cs[e]) { ok = false; break; }
    }
    if (ok) leaf(c, ce, combo);
  }
}

// order-preserving map double -> uint64 (larger score <=> larger key); NaN maps below -inf
TW_HD unsigned long long score_key(double s) {
  if (s != s) return 0ULL;
  unsigned long long u;
#if defined(__CUDA_ARCH__)
  u = (unsigned long long)__double_as_longlong(s);
#else
  memcpy(&u, &s, sizeof u);
#endif
  return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}

// total order used when partial top-K lists are merged: the reference's (score, stack) order and,
// where that order calls two tuples equal, the earlier DFS leaf first (what a single sequential
// enumeration with topk_offer produces)
TW_HD bool cand_ahead(const ProbView& v, double sa, const int* ca, double sb, const int* cb) {
  if (cand_less(v, sb, cb, sa, ca)) return true;
  if (cand_less(v, sa, ca, sb, cb)) return false;
  for (int e = 0; e < v.E; ++e)
    if (ca[e] != cb[e]) return ca[e] < cb[e];
  return false;
}

// first index in [0, n) of a sorted array with a[idx] >= key
TW_HD int lower_bound(const int64_t* a, int n, int64_t key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}
// first index with a[idx] > key
TW_HD int upper_bound(const int64_t* a, int n, int64_t key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (key < a[mid]) hi = mid; else lo = mid + 1;
  }
  return lo;
}
// lower_bound knowing the answer is >= from (galloping; in-spans arrive sorted by start)
TW_HD int lower_bound_from(const int64_t* a, int n, int from, int64_t key) {
  if (from >= n || a[from] >= key) return from;
  int step = 1, lo = from, hi = from + 1;
  while (hi < n && a[hi] < key) { lo = hi; step <<= 1; hi = lo + step; }
  if (hi > n) hi = n;
  // invariant: a[lo] < key, (hi == n or a[hi] >= key)
  ++lo;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// ---------------------------------------------------------------------------------------------
// PerfectCut (V3:1024-1039) support: "used" bitmaps.  Bit j of ep e <=> out span lo_e + j appears
// in some feasible tuple of the in-span (candidates_array, V3:1043-1051).
// ---------------------------------------------------------------------------------------------
// any common set bit between A (origin loA) and B (origin loB >= loA), both W words
TW_HD bool bitmaps_intersect(const uint32_t* A, int loA, const uint32_t* B, int loB, int W) {
  int shift = loB - loA;           // >= 0: in-spans are sorted by start
  if (shift < 0) {                 // defensive: swap roles
    const uint32_t* t = A; A = B; B = t; shift = -shift;
  }
  int ws = shift >> 5, bs = shift & 31;
  for (int wi = 0; wi < W; ++wi) {
    int ai = wi + ws;
    if (ai >= W) break;
    uint32_t a = A[ai] >> bs;
    if (bs && ai + 1 < W) a |= A[ai + 1] << (32 - bs);
    if (a & B[wi]) return true;
  }
  return false;
}

// ---------------------------------------------------------------------------------------------
// Per-window stitch: BuildMISInstance (V3:1252-1274) + exact MWIS (gurobi_optimods.mwis at
// V3:1411).  Vertices are (in-span k, rank r) with weight 10000 + score; two vertices conflict
// when they belong to the same in-span or share an out span at the same tuple position
// (AssignmentIntersect, V3:1276-1281).  Because every in-span's candidates form a clique, an
// independent set picks at most one rank per in-span: branch and bound over in-spans ("rank r or
// none"), after splitting the window into connected components of the in-span conflict graph.
// Vertices with weight <= 0 are never taken (score < -10000, SURVEY A.9 item 6).
// ---------------------------------------------------------------------------------------------
// The window functions below take either buffer type; they reach tuple position e of candidate
// (in-span k, rank r) only through at(k, r, e).
struct WindowBuf {
  double score[TW_WINDOW_CAP][TW_K];
  int idx[TW_WINDOW_CAP][TW_K][TW_MAX_E];
  int cnt[TW_WINDOW_CAP];
  int chosen[TW_WINDOW_CAP];
  uint32_t adj[TW_WINDOW_CAP];
  TW_HD int& at(int k, int r, int e) { return idx[k][r][e]; }
  TW_HD int at(int k, int r, int e) const { return idx[k][r][e]; }
};

// The window buffer of the stitch kernel: one plane of candidates per tuple position, the last member,
// so a holder may provide only packed_bytes(E_max) bytes, the planes of its largest E (the stitch
// kernel's per-warp slab, sized per batch).  Lane 5k + r reading (k, r) hits 32 distinct banks.
struct PackedWindowBuf {
  double score[TW_WINDOW_CAP][TW_K];
  int cnt[TW_WINDOW_CAP];
  int chosen[TW_WINDOW_CAP];
  uint32_t adj[TW_WINDOW_CAP];
  int idx[TW_MAX_E][TW_WINDOW_CAP * TW_K];
  TW_HD int& at(int k, int r, int e) { return idx[e][k * TW_K + r]; }
  TW_HD int at(int k, int r, int e) const { return idx[e][k * TW_K + r]; }
  static constexpr int packed_bytes(int e_max) {
    return (int)(sizeof(PackedWindowBuf) - sizeof(int) * TW_WINDOW_CAP * TW_K * (TW_MAX_E - e_max));
  }
};

TW_HD bool tuples_conflict(const int* a, const int* b, int E) {
  for (int e = 0; e < E; ++e)
    if (a[e] == b[e]) return true;
  return false;
}

// candidates (k, r) and (a, q) of a window share an out span at some tuple position
template <class WB>
TW_HD bool cands_conflict(const WB& wb, int k, int r, int a, int q, int E) {
  for (int e = 0; e < E; ++e)
    if (wb.at(k, r, e) == wb.at(a, q, e)) return true;
  return false;
}

// in-span level adjacency: bit a of adj[k] <=> some candidate of k conflicts with some of a
template <class WB>
TW_HD uint32_t window_adjacency(const WB& wb, int E, int nw, int k) {
  uint32_t m = 0;
  for (int a = 0; a < nw; ++a) {
    if (a == k) continue;
    bool hit = false;
    for (int r = 0; r < wb.cnt[k] && !hit; ++r)
      for (int q = 0; q < wb.cnt[a] && !hit; ++q)
        hit = cands_conflict(wb, k, r, a, q, E);
    if (hit) m |= 1u << a;
  }
  return m;
}

// E == 1: a candidate is one out span, so a connected component of the window is a maximum-weight
// bipartite matching (in-spans x out spans, at most one edge per candidate, an in-span may stay
// unmatched at weight 0).  Solved exactly in polynomial time by the Hungarian method (shortest
// augmenting paths with potentials, sparse rows: <= 5 candidates + one private "unassigned"
// column per in-span) instead of branch and bound, whose search explodes when ~30 in-spans compete
// for interchangeable spans.  Same optimum as the MWIS formulation of V3:1252-1274.
#define TW_ASSIGN_MAX_COLS (TW_WINDOW_CAP * (TW_K + 1) + 1)
constexpr int kMwisPricedMin = 7;   // components of at least this many in-spans get the priced bound
constexpr int kMwisSimpleBudget = 1024;   // nodes the plain search may spend on a component before the priced one takes over
// `pos`: tuple position whose spans are the columns (E = 1: position 0 is the whole problem; E > 1: the
// projection of the window on one callee, a RELAXATION whose dual prices bound the branch and bound
// below).  best != nullptr: the matching (first tied optimum); price != nullptr: the dual price of
// every candidate's column and their total (a candidate's weight never exceeds its row's dual plus
// its column's price; prices are >= 0).
template <class WB>
TW_HD_NOINLINE inline void assignment_solve(const WB& wb, const int* member, int m, int pos, int* best,
                                            double (*price)[TW_K], double* price_total) {
  // columns 1..ncol: distinct out spans; ncol+1..ncol+m: "row l stays unassigned"
  int colid[TW_WINDOW_CAP * TW_K];
  int ncol = 0;
  short ecol[TW_WINDOW_CAP][TW_K];
  for (int l = 0; l < m; ++l) {
    const int k = member[l];
    for (int r = 0; r < TW_K; ++r) {
      ecol[l][r] = -1;
      if (r >= wb.cnt[k] || !(TW_WEIGHT_OFFSET + wb.score[k][r] > 0.0)) continue;
      const int span = wb.at(k, r, pos);
      int j = 0;
      while (j < ncol && colid[j] != span) ++j;
      if (j == ncol) colid[ncol++] = span;
      ecol[l][r] = (short)(j + 1);
    }
  }
  const int M = ncol + m;
  double u[TW_WINDOW_CAP + 1], vv[TW_ASSIGN_MAX_COLS], minv[TW_ASSIGN_MAX_COLS];
  short p[TW_ASSIGN_MAX_COLS], way[TW_ASSIGN_MAX_COLS];
  bool used[TW_ASSIGN_MAX_COLS];
  for (int i = 0; i <= m; ++i) u[i] = 0.0;
  for (int j = 0; j <= M; ++j) { vv[j] = 0.0; p[j] = 0; way[j] = 0; }
  const double INF = 1e300;
  for (int i = 1; i <= m; ++i) {
    p[0] = (short)i;
    int j0 = 0;
    for (int j = 0; j <= M; ++j) { minv[j] = INF; used[j] = false; }
    do {
      used[j0] = true;
      const int i0 = p[j0], l0 = i0 - 1, k0 = member[l0];
      // relax the (sparse) row i0: its candidates cost -(10000 + score), its private column 0
      for (int r = 0; r <= TW_K; ++r) {
        int j;
        double c;
        if (r < TW_K) {
          j = ecol[l0][r];
          if (j < 0) continue;
          c = -(TW_WEIGHT_OFFSET + wb.score[k0][r]);
        } else {
          j = ncol + i0;
          c = 0.0;
        }
        if (used[j]) continue;
        const double cur = c - u[i0] - vv[j];
        if (cur < minv[j]) { minv[j] = cur; way[j] = (short)j0; }
      }
      double delta = INF;
      int j1 = 0;
      for (int j = 1; j <= M; ++j)
        if (!used[j] && minv[j] < delta) { delta = minv[j]; j1 = j; }
      for (int j = 0; j <= M; ++j) {
        if (used[j]) { u[p[j]] += delta; vv[j] -= delta; }
        else if (minv[j] < INF) minv[j] -= delta;
      }
      j0 = j1;
    } while (p[j0] != 0);
    do {
      const int j1 = way[j0];
      p[j0] = p[j1];
      j0 = j1;
    } while (j0);
  }
  if (price) {
    double tot = 0.0;
    for (int j = 1; j <= ncol; ++j) tot += -vv[j];
    *price_total = tot;
    for (int l = 0; l < m; ++l)
      for (int r = 0; r < TW_K; ++r) price[l][r] = ecol[l][r] >= 1 ? -vv[ecol[l][r]] : 0.0;
  }
  if (!best) return;
  // ---- tied optima (TW_MWIS_TIE_TOL): the canonical answer is the FIRST optimal solution in the
  // depth-first order of the branch and bound (in-spans ascending; ranks ascending, "unassigned"
  // last).  Every optimal matching lives in the equality subgraph of the final potentials (edges
  // with zero reduced cost), so: fix the rows in order; a row takes its first tight option for which
  // the remaining rows can still be matched along tight edges (one alternating-path search).  With no
  // ties the only tight option is the matched one and this pass is O(m).
  short rowcol[TW_WINDOW_CAP];
  for (int l = 0; l < m; ++l) rowcol[l] = 0;
  for (int j = 1; j <= M; ++j)
    if (p[j] != 0) rowcol[p[j] - 1] = (short)j;
  bool fixedc[TW_ASSIGN_MAX_COLS];
  for (int j = 0; j <= M; ++j) fixedc[j] = false;
  auto opt_col = [&](int l, int r) { return r < TW_K ? (int)ecol[l][r] : ncol + 1 + l; };
  auto tight = [&](int l, int r) {
    const int j = opt_col(l, r);
    if (j < 0) return false;
    const double c = r < TW_K ? -(TW_WEIGHT_OFFSET + wb.score[member[l]][r]) : 0.0;
    return c - u[l + 1] - vv[j] <= TW_MWIS_TIE_TOL;
  };
  for (int l = 0; l < m; ++l) best[l] = -1;
  for (int l = 0; l < m; ++l) {
    for (int r = 0; r <= TW_K; ++r) {
      if (!tight(l, r)) continue;
      const int j = opt_col(l, r);
      if (fixedc[j]) continue;
      bool ok = rowcol[l] == j;
      if (!ok) {
        const int owner = p[j] - 1;               // row holding column j now (-1: free); never a fixed row
        const int freed = rowcol[l];
        if (owner < 0) {
          p[freed] = 0; p[j] = (short)(l + 1); rowcol[l] = (short)j;
          ok = true;
        } else {
          // re-match `owner` along tight edges: columns j and the fixed ones are closed, `freed` is free
          short st_row[TW_WINDOW_CAP + 1], st_opt[TW_WINDOW_CAP + 1], st_col[TW_WINDOW_CAP + 1];
          for (int q = 0; q <= M; ++q) used[q] = fixedc[q];
          used[j] = true;
          p[freed] = 0;
          int depth = 0;
          st_row[0] = (short)owner; st_opt[0] = 0;
          bool found = false;
          while (depth >= 0 && !found) {
            const int x = st_row[depth];
            bool pushed = false;
            while (st_opt[depth] <= TW_K) {
              const int rr = st_opt[depth]++;
              if (!tight(x, rr)) continue;
              const int jj = opt_col(x, rr);
              if (used[jj]) continue;
              used[jj] = true;
              st_col[depth] = (short)jj;
              if (p[jj] == 0) { found = true; break; }
              st_row[depth + 1] = (short)(p[jj] - 1);
              st_opt[depth + 1] = 0;
              ++depth;
              pushed = true;
              break;
            }
            if (found) break;
            if (!pushed) --depth;
          }
          if (found) {
            for (int d = depth; d >= 0; --d) {     // shift every row on the path to its new column
              const int x = st_row[d], jj = st_col[d];
              p[jj] = (short)(x + 1);
              rowcol[x] = (short)jj;
            }
            p[j] = (short)(l + 1);
            rowcol[l] = (short)j;
            ok = true;
          } else {
            p[freed] = (short)(l + 1);             // nothing was changed: restore
          }
        }
      }
      if (ok) {
        fixedc[j] = true;
        best[l] = r < TW_K ? r : -1;
        break;
      }
    }
  }
}

// Solves the window; wb.adj must be filled.  Returns the number of search nodes, or -1 when
// node_limit is exceeded (TW_ERR_MWIS_LIMIT).
// `deferred` (device callers): components whose plain search ran out of its budget are not searched
// here but returned as in-span masks (up to TW_MWIS_MAX_DEFERRED; *n_deferred counts them) for the
// caller's warp-wide priced search (tw_stitch.cu); nullptr: everything is solved here.
#define TW_MWIS_MAX_DEFERRED 4
template <class WB>
TW_HD_NOINLINE inline long long mwis_solve(WB& wb, int E, int nw, long long node_limit,
                                           uint32_t* deferred = nullptr, int* n_deferred = nullptr) {
  long long nodes = 0;
  if (n_deferred) *n_deferred = 0;
  uint32_t todo = nw >= 32 ? 0xffffffffu : ((1u << nw) - 1u);
  for (int k = 0; k < nw; ++k) wb.chosen[k] = -1;
  while (todo) {
    // connected component of the lowest remaining in-span
    int seed = 0;
    while (!(todo >> seed & 1u)) ++seed;
    uint32_t comp = 1u << seed, frontier = comp;
    while (frontier) {
      int k = 0;
      while (!(frontier >> k & 1u)) ++k;
      frontier &= ~(1u << k);
      uint32_t nb = wb.adj[k] & ~comp;
      comp |= nb;
      frontier |= nb;
    }
    todo &= ~comp;
    int member[TW_WINDOW_CAP];
    int m = 0;
    for (int k = 0; k < nw; ++k)
      if (comp >> k & 1u) member[m++] = k;
    if (m == 1) {  // isolated in-span: its best candidate, if the weight is positive
      int k = member[0];
      if (wb.cnt[k] > 0 && TW_WEIGHT_OFFSET + wb.score[k][0] > 0.0) wb.chosen[k] = 0;
      ++nodes;
      continue;
    }
    if (E == 1 && m >= 3) {   // bipartite case: exact matching in polynomial time
      int bst[TW_WINDOW_CAP];
      assignment_solve(wb, member, m, 0, bst, nullptr, nullptr);
      for (int l = 0; l < m; ++l) wb.chosen[member[l]] = bst[l];
      nodes += m;
      continue;
    }
    // Two searches with the same answer (the first tied optimum in depth-first order): a plain one with
    // the static bound "sum of the remaining in-spans' best weights" — a few instructions per node,
    // enough for almost every window — and, when that one runs out of its small node budget, the
    // search with availability masks and dual prices below (tens of times fewer nodes on windows
    // whose in-spans compete for interchangeable spans, several times the work per node).
    bool simple_done = true;
    const long long nodes_at_start = nodes;
    {
      double ub[TW_WINDOW_CAP + 1];
      ub[m] = 0.0;
      for (int l = m - 1; l >= 0; --l) {
        int k = member[l];
        double mx = 0.0;
        for (int r = 0; r < wb.cnt[k]; ++r) {
          double w = TW_WEIGHT_OFFSET + wb.score[k][r];
          if (w > mx) mx = w;
        }
        ub[l] = ub[l + 1] + mx;
      }
      int choice[TW_WINDOW_CAP], best[TW_WINDOW_CAP], iter[TW_WINDOW_CAP + 1];
      double cur[TW_WINDOW_CAP + 1];
      double best_w = -1.0;
      for (int l = 0; l < m; ++l) best[l] = -1;
      int level = 0;
      cur[0] = 0.0;
      iter[0] = 0;
      while (level >= 0) {
        if (level == m) {
          ++nodes;
          if (cur[m] > best_w + TW_MWIS_TIE_TOL) {   // a tied total never replaces an earlier leaf
            best_w = cur[m];
            for (int l = 0; l < m; ++l) best[l] = choice[l];
          }
          --level;
          continue;
        }
        int k = member[level];
        if (iter[level] == 0) {
          ++nodes;
          if (nodes - nodes_at_start > kMwisSimpleBudget) { simple_done = false; break; }
          if (cur[level] + ub[level] <= best_w + TW_MWIS_TIE_TOL) { --level; continue; }
        }
        int r = iter[level]++;
        if (r > wb.cnt[k]) { --level; continue; }
        if (r == wb.cnt[k]) {  // leave in-span k unassigned
          choice[level] = -1;
          cur[level + 1] = cur[level];
          ++level;
          iter[level] = 0;
          continue;
        }
        double w = TW_WEIGHT_OFFSET + wb.score[k][r];
        if (!(w > 0.0)) continue;
        bool ok = true;
        for (int l = 0; l < level && ok; ++l)
          if (choice[l] >= 0 && (wb.adj[k] >> member[l] & 1u) &&
              cands_conflict(wb, k, r, member[l], choice[l], E))
            ok = false;
        if (!ok) continue;
        choice[level] = r;
        cur[level + 1] = cur[level] + w;
        ++level;
        iter[level] = 0;
      }

      if (simple_done) {
        for (int l = 0; l < m; ++l) wb.chosen[member[l]] = best[l];
        continue;
      }
    }
    // (a component that exhausts the plain budget has many in-spans; a window of <= 31 in-spans
    // cannot hold more than TW_MWIS_MAX_DEFERRED of them, so the list cannot overflow)
    if (deferred && *n_deferred < TW_MWIS_MAX_DEFERRED) {
      deferred[(*n_deferred)++] = comp;
      continue;
    }
#ifdef __CUDA_ARCH__
    return -1;   // device callers always pass `deferred`: the sequential priced search is host-only
#else
    // Depth-first branch and bound over the component's in-spans in window order ("rank r", ranks
    // ascending, then "unassigned").  avail[L][j] = ranks of in-span j (j >= L) that are still
    // compatible with the choices made at levels < L; the bound of a node is the sum over the
    // remaining in-spans of their best AVAILABLE weight (lists are sorted by score, so that is the
    // lowest available rank).  Compared with the static sum of maxima this cuts the search of windows
    // in which ~30 in-spans compete for interchangeable spans by orders of magnitude; the optimum and
    // the tie rule (first tied leaf in this order, TW_MWIS_TIE_TOL) are unchanged.
    uint8_t avail[TW_WINDOW_CAP + 1][TW_WINDOW_CAP];
    double rem[TW_WINDOW_CAP + 1];                 // plain bound of the in-spans L..m-1 given avail[L]
    // Large components: second bound from the dual prices of ONE callee's assignment relaxation (every
    // out span of that callee serves at most one in-span): sum over the remaining in-spans of their
    // best available REDUCED weight (weight - price of its span, floored at 0) + the prices not yet
    // spent.  At the root this equals the relaxation's optimum — far below the sum of maxima when the
    // in-spans compete for the same spans — and it stays valid at every node for any prices >= 0.
    double price[TW_WINDOW_CAP][TW_K];
    double remp[TW_WINDOW_CAP + 1], lam[TW_WINDOW_CAP + 1];
    const bool priced = m >= kMwisPricedMin;
    if (priced) {
      int pos = 0, fewest = 0x7fffffff;           // the callee with the fewest distinct spans: most competition
      for (int e = 0; e < E; ++e) {
        int distinct = 0;
        for (int l = 0; l < m; ++l)
          for (int r = 0; r < wb.cnt[member[l]]; ++r) {
            const int sp = wb.at(member[l], r, e);
            bool seen = false;
            for (int l2 = 0; l2 <= l && !seen; ++l2)
              for (int r2 = 0; r2 < (l2 < l ? wb.cnt[member[l2]] : r) && !seen; ++r2)
                seen = wb.at(member[l2], r2, e) == sp;
            distinct += !seen;
          }
        if (distinct < fewest) { fewest = distinct; pos = e; }
      }
      assignment_solve(wb, member, m, pos, nullptr, price, &lam[0]);
      nodes += m;
    } else {
      lam[0] = 0.0;
      for (int l = 0; l < m; ++l)
        for (int r = 0; r < TW_K; ++r) price[l][r] = 0.0;
    }
    auto best_avail = [&](int j, uint8_t mask) {
      if (!mask) return 0.0;
      int r = 0;
      while (!(mask >> r & 1u)) ++r;
      return TW_WEIGHT_OFFSET + wb.score[member[j]][r];
    };
    auto best_reduced = [&](int j, uint8_t mask) {
      double mx = 0.0;
      for (int r = 0; r < TW_K; ++r)
        if (mask >> r & 1u) {
          const double v = TW_WEIGHT_OFFSET + wb.score[member[j]][r] - price[j][r];
          mx = v > mx ? v : mx;
        }
      return mx;
    };
    rem[0] = 0.0;
    remp[0] = 0.0;
    for (int l = 0; l < m; ++l) {
      const int k = member[l];
      uint8_t mask = 0;
      for (int r = 0; r < wb.cnt[k]; ++r)
        if (TW_WEIGHT_OFFSET + wb.score[k][r] > 0.0) mask |= (uint8_t)(1u << r);
      avail[0][l] = mask;
    }
    for (int l = m - 1; l >= 0; --l) {
      rem[0] += best_avail(l, avail[0][l]);
      remp[0] += best_reduced(l, avail[0][l]);
    }
    int choice[TW_WINDOW_CAP], best[TW_WINDOW_CAP], iter[TW_WINDOW_CAP + 1];
    double cur[TW_WINDOW_CAP + 1];
    double best_w = -1.0;
    for (int l = 0; l < m; ++l) best[l] = -1;
    int level = 0;
    cur[0] = 0.0;
    iter[0] = 0;
    while (level >= 0) {
      if (level == m) {
        ++nodes;
        if (cur[m] > best_w + TW_MWIS_TIE_TOL) {   // a tied total never replaces an earlier leaf
          best_w = cur[m];
          for (int l = 0; l < m; ++l) best[l] = choice[l];
        }
        --level;
        continue;
      }
      const int k = member[level];
      if (iter[level] == 0) {
        ++nodes;
        if (node_limit > 0 && nodes > node_limit) return -1;
        double bound = rem[level];
        if (priced) {
          // (a few ulps of slack: the priced bound is assembled from differences of large numbers)
          const double bp = remp[level] + lam[level] + 1e-7;
          bound = bp < bound ? bp : bound;
        }
        if (cur[level] + bound <= best_w + TW_MWIS_TIE_TOL) { --level; continue; }
      }
      const int r = iter[level]++;
      if (r > wb.cnt[k]) { --level; continue; }
      if (r == wb.cnt[k]) {  // leave in-span k unassigned
        choice[level] = -1;
        cur[level + 1] = cur[level];
        for (int j = level + 1; j < m; ++j) avail[level + 1][j] = avail[level][j];
        rem[level + 1] = rem[level] - best_avail(level, avail[level][level]);
        remp[level + 1] = remp[level] - best_reduced(level, avail[level][level]);
        lam[level + 1] = lam[level];
        ++level;
        iter[level] = 0;
        continue;
      }
      if (!(avail[level][level] >> r & 1u)) continue;      // weight <= 0, or taken by an earlier choice
      const double w = TW_WEIGHT_OFFSET + wb.score[k][r];
      // the choice closes the conflicting ranks of the later in-spans
      double rest = 0.0, restp = 0.0;
      for (int j = level + 1; j < m; ++j) {
        uint8_t mask = avail[level][j];
        if (mask && (wb.adj[k] >> member[j] & 1u)) {
          const int kj = member[j];
          for (int q = 0; q < wb.cnt[kj]; ++q)
            if ((mask >> q & 1u) && cands_conflict(wb, k, r, kj, q, E)) mask &= (uint8_t)~(1u << q);
        }
        avail[level + 1][j] = mask;
        rest += best_avail(j, mask);
        if (priced) restp += best_reduced(j, mask);
      }
      choice[level] = r;
      cur[level + 1] = cur[level] + w;
      rem[level + 1] = rest;
      remp[level + 1] = restp;
      lam[level + 1] = lam[level] - price[level][r];
      ++level;
      iter[level] = 0;
    }
    for (int l = 0; l < m; ++l) wb.chosen[member[l]] = best[l];
#endif
  }
  return nodes;
}

// ---------------------------------------------------------------------------------------------
// Windows from cut flags: CreateWindows2's loop, V3:1056-1076, as a cursor the stitch kernel
// advances once per in-span.  cut[i] = PerfectCut(i) for 1 <= i <= n-2 and 0 elsewhere.
//   visit n-1                          -> window ends at n-1
//   visit i, cut[i]                    -> window ended at i-1 (seen here as look-ahead), count = 0
//   visit i, else current_count == 30  -> window ends at i, count = 0
// A window that starts at a perfect cut can hold 31 in-spans (the count restarts at 0 there,
// at 1 after a size cut): TW_WINDOW_CAP.
// ---------------------------------------------------------------------------------------------
struct WindowCursor {
  int count;
  TW_HD void init() { count = 1; }
  TW_HD bool ends_at(int i, int n, const uint8_t* cut) {
    if (i == n - 1) return i != 0;
    bool end = false;
    if (i != 0) {
      if (cut[i]) count = 0;
      else if (count == TW_MAX_WINDOW) { count = 0; end = true; }
    }
    count += 1;
    if (cut[i + 1]) end = true;
    return end;
  }
};

}  // namespace tw
