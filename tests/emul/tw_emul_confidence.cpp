// tw_emul_confidence.cpp — CPU stepping of the request confidence (tw_confidence.cu).
//
// TEST INFRASTRUCTURE ONLY, like tw_emul.cpp: the per-in-span step (conf_choice), its exp and log and the
// per-request confidence (conf_request) are the kernels' own functions in tw_core.cuh, compiled with g++.
// Written for the CPU: the threads as a loop over in-spans, the atomics as plain adds and a running min,
// and the sums in the kernels' fixed order (256 threads, a butterfly per warp, the warps in order).  The
// roots come in from the caller (the join is tw_traces.cu's, tested on its own).
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../traceweaver_b200/csrc/tw_core.cuh"

using namespace tw;

// tree_cta_sum (tw_kernels.cuh) over v[0 .. n)
static double cta_sum(const double* v, int64_t n) {
  double lane[256] = {0.0}, y[32];
  for (int t = 0; t < 256; ++t)
    for (int64_t x = t; x < n; x += 256) lane[t] = dadd(lane[t], v[x]);
  for (int w = 0; w < 8; ++w) {
    double* l = lane + 32 * w;
    for (int d = 16; d > 0; d >>= 1) {
      for (int k = 0; k < 32; ++k) y[k] = dadd(l[k], l[k ^ d]);
      memcpy(l, y, sizeof y);
    }
  }
  double s = lane[0];
  for (int w = 1; w < 8; ++w) s = dadd(s, lane[32 * w]);
  return s;
}

extern "C" void twe_conf_exp(int64_t n, const double* d, double* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = conf_exp(d[i]);
}

extern "C" void twe_conf_log(int64_t n, const double* x, double* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = conf_log(x[i]);
}

// q: the fixed-point ell of every in-span (-1 where p == 0).  Returns TW_ERR_RANGE_LIMIT for a request of
// TW_CONF_MAX_DECISIONS or more decisions.
extern "C" int twe_request_confidence(const tw_batch* b, const int32_t* assign, const int32_t* root,
                                      const double* score, const uint8_t* code, const double* topk_score,
                                      const int32_t* topk_idx, const uint8_t* topk_cnt, double* p, double* ell,
                                      int64_t* q, int32_t* decisions, int32_t* zero, int64_t* log_conf, double* conf,
                                      int32_t* weakest, double* weakest_p, double* est_accuracy, int32_t* requests,
                                      double* expected_exact) {
  const int64_t n_in = b->n_in_total;
  const int P = b->n_problems;
  std::vector<uint64_t> wbits((size_t)n_in, ~0ULL);
  for (int64_t x = 0; x < n_in; ++x) {
    decisions[x] = zero[x] = 0;
    log_conf[x] = 0;
  }
  for (int pb = 0; pb < P; ++pb) {
    const int64_t in0 = b->prob_in_off[pb], n = b->prob_in_off[pb + 1] - in0;
    const int E = b->prob_ep_off[pb + 1] - b->prob_ep_off[pb];
    const int64_t tup = b->prob_tuple_off[pb];
    for (int64_t i = 0; i < n; ++i) {
      const int64_t g = in0 + i;
      int32_t c[TW_MAX_E];
      for (int e = 0; e < E; ++e) c[e] = assign[tup + e * n + i];
      const ConfChoice ch = conf_choice(E, c, code[g], score[g], topk_score + g * TW_K,
                                        topk_idx + TW_K * (tup + i * E), topk_cnt[g]);
      p[g] = ch.p;
      ell[g] = ch.ell;
      q[g] = ch.q;
    }
  }
  for (int64_t g = 0; g < n_in; ++g) {
    const int32_t r = root[g];
    weakest[g] = r == g ? 0x7fffffff : -1;
    if (r < 0 || r >= n_in) continue;
    decisions[r] += 1;
    if (q[g] < 0) zero[r] += 1;
    else log_conf[r] += q[g];
    if (conf_bits(p[g]) < wbits[(size_t)r]) wbits[(size_t)r] = conf_bits(p[g]);
  }
  int rc = TW_OK;
  for (int64_t g = 0; g < n_in; ++g) {
    const int32_t r = root[g];
    if (r >= 0 && r < n_in && conf_bits(p[g]) == wbits[(size_t)r] && g < weakest[r]) weakest[r] = (int32_t)g;
    if (r != g) {
      conf[g] = weakest_p[g] = tw_nan();
      continue;
    }
    conf[g] = conf_request(log_conf[g], zero[g]);
    weakest_p[g] = conf_from_bits(wbits[(size_t)g]);
    if (decisions[g] >= TW_CONF_MAX_DECISIONS) rc = TW_ERR_RANGE_LIMIT;
  }
  std::vector<double> seg((size_t)P), roots;
  int32_t nreq = 0;
  for (int pb = 0; pb < P; ++pb) {
    const int64_t lo = b->prob_in_off[pb], hi = b->prob_in_off[pb + 1];
    est_accuracy[pb] = ddiv(cta_sum(p + lo, hi - lo), (double)(hi - lo));
    roots.assign((size_t)(hi - lo), 0.0);
    for (int64_t x = lo; x < hi; ++x)
      if (root[x] == x) {
        roots[(size_t)(x - lo)] = conf[x];
        ++nreq;
      }
    seg[(size_t)pb] = cta_sum(roots.data(), hi - lo);
  }
  requests[0] = nreq;
  expected_exact[0] = cta_sum(seg.data(), P);
  return rc;
}
