// tw_emul_critical.cpp — CPU stepping of the critical-path walk (tw_critical_path.cu).
//
// TEST INFRASTRUCTURE ONLY, like tw_emul.cpp: the per-node steps and the last level's walk are the
// kernels' own functions (cp_in_span_step, cp_out_span_step, cp_tail_walk in tw_core.cuh), compiled with
// g++.  Written for the CPU: the level loop (one launch per level in the kernels), the threads of a level
// as a loop over in-spans, the culprit as a running max / min, and the sums in node order.  The roots come
// in from the caller (the join is tw_traces.cu's, tested on its own).
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../traceweaver_b200/csrc/tw_core.cuh"

using namespace tw;

template <class T>
struct Walk {
  const tw_batch& b;
  const T *in_s, *in_e, *out_s, *out_e;
  const int32_t *assign, *in_caller;
  uint8_t* on_path;
  double* self_us;
  std::vector<int32_t> claim, owner, level;     // out-span -> its callee in-span / the in-span that took it
  std::vector<T> wlo, whi;
  std::vector<int> prob;

  // k_cp_level's visit: in-span x with its window; the callee in-spans it puts on the path get level `mark`
  int visit(int64_t x, int mark) {
    const int64_t n_in = b.n_in_total;
    const int p = prob[(size_t)x];
    const int64_t in0 = b.prob_in_off[p], n = b.prob_in_off[p + 1] - in0, i = x - in0;
    const int ep0 = b.prob_ep_off[p], E = b.prob_ep_off[p + 1] - ep0;
    bool has[TW_MAX_E], on[TW_MAX_E];
    T cs[TW_MAX_E], ce[TW_MAX_E], lo[TW_MAX_E], hi[TW_MAX_E];
    int64_t k[TW_MAX_E];
    for (int e = 0; e < E; ++e) {
      const int32_t j = assign[b.prob_tuple_off[p] + e * n + i];
      has[e] = j >= 0;
      k[e] = has[e] ? b.ep_out_off[ep0 + e] + j : 0;
      cs[e] = has[e] ? out_s[k[e]] : T(0);
      ce[e] = has[e] ? out_e[k[e]] : T(0);
    }
    const T self = cp_in_span_step<T>(E, has, cs, ce, wlo[(size_t)x], whi[(size_t)x], on, lo, hi);
    on_path[x] = 1;
    self_us[x] = (double)self;
    int m = 0;
    for (int e = 0; e < E; ++e) {
      if (!on[e]) continue;
      const int32_t y = claim[(size_t)k[e]];
      bool y_on = false;
      T ylo = 0, yhi = 0;
      const T ks = cp_out_span_step<T>(lo[e], hi[e], y >= 0, y >= 0 ? in_s[y] : T(0), y >= 0 ? in_e[y] : T(0),
                                       &y_on, &ylo, &yhi);
      on_path[n_in + k[e]] = 1;
      self_us[n_in + k[e]] = (double)ks;
      if (y_on) {
        wlo[(size_t)y] = ylo;
        whi[(size_t)y] = yhi;
        level[(size_t)y] = mark;
        ++m;
      }
    }
    return m;
  }
};

// The tree below the last level for cp_tail_walk, as the kernel's CpTail reads it
template <class T>
struct Tail {
  Walk<T>& w;
  int mark;
  int64_t tup = 0, n = 0, i = 0;
  int ep0 = 0;

  int enter(int32_t y) {
    const int p = w.prob[(size_t)y];
    tup = w.b.prob_tuple_off[p];
    n = w.b.prob_in_off[p + 1] - w.b.prob_in_off[p];
    i = y - w.b.prob_in_off[p];
    ep0 = w.b.prob_ep_off[p];
    return w.b.prob_ep_off[p + 1] - ep0;
  }
  int32_t child(int e) const {
    const int32_t j = w.assign[tup + e * n + i];
    if (j < 0) return -1;
    const int32_t y = w.claim[(size_t)(w.b.ep_out_off[ep0 + e] + j)];
    return y >= 0 && w.level[(size_t)y] == mark ? y : -1;
  }
  void visit(int32_t y) { w.visit(y, mark); }
  int32_t up(int32_t y, int* e) const {
    const int64_t k = w.in_caller[y] - w.b.n_in_total;
    const int32_t x = w.owner[(size_t)k];
    const int p = w.prob[(size_t)x];
    int ep = w.b.prob_ep_off[p];
    while (w.b.ep_out_off[ep + 1] <= k) ++ep;
    *e = ep - w.b.prob_ep_off[p];
    return x;
  }
};

template <class T>
static void walk(const tw_batch& b, const T* in_s, const T* in_e, const T* out_s, const T* out_e,
                 const int32_t* assign, const int32_t* in_caller, const int32_t* root, double slow_us, int levels,
                 uint8_t* on_path, double* self_us, int32_t* culprit, double* server_us, int32_t* server_visits,
                 double* call_us, int32_t* requests) {
  const int64_t n_in = b.n_in_total, n_out = b.n_out_total, N = n_in + n_out;
  const int P = b.n_problems;
  Walk<T> w{b, in_s, in_e, out_s, out_e, assign, in_caller, on_path, self_us};
  w.claim.assign((size_t)n_out, -1);
  w.owner.assign((size_t)n_out, -1);
  w.level.assign((size_t)n_in, -1);
  w.wlo.resize((size_t)n_in);
  w.whi.resize((size_t)n_in);
  w.prob.resize((size_t)n_in);
  for (int64_t y = 0; y < n_in; ++y)
    if (in_caller[y] >= 0) w.claim[(size_t)(in_caller[y] - n_in)] = (int32_t)y;
  for (int p = 0; p < P; ++p) {
    const int64_t in0 = b.prob_in_off[p], n = b.prob_in_off[p + 1] - in0;
    for (int64_t x = in0; x < b.prob_in_off[p + 1]; ++x) w.prob[(size_t)x] = p;
    for (int e = 0; e < b.prob_ep_off[p + 1] - b.prob_ep_off[p]; ++e)
      for (int64_t i = 0; i < n; ++i) {
        const int32_t j = assign[b.prob_tuple_off[p] + e * n + i];
        if (j >= 0) w.owner[(size_t)(b.ep_out_off[b.prob_ep_off[p] + e] + j)] = (int32_t)(in0 + i);
      }
  }
  std::vector<uint8_t> slow((size_t)n_in, 0);
  memset(on_path, 0, (size_t)N);
  for (int64_t x = 0; x < N; ++x) self_us[x] = 0.0;
  requests[0] = requests[1] = 0;
  for (int64_t x = 0; x < n_in; ++x) {
    culprit[x] = -1;
    if (root[x] != x) continue;
    const T a = in_s[x], e = in_e[x], bb = e > a ? e : a;
    w.wlo[(size_t)x] = a;
    w.whi[(size_t)x] = bb;
    w.level[(size_t)x] = 0;
    slow[(size_t)x] = (double)(bb - a) >= slow_us;
    requests[0] += 1;
    requests[1] += slow[(size_t)x];
  }
  // levels 0 .. levels - 1, the last of them walking what lies below it; levels <= 0: until nothing is left
  for (int L = 0; levels <= 0 || L < levels; ++L) {
    const bool last = L == levels - 1;
    bool activated = false;
    for (int64_t x = 0; x < n_in; ++x) {
      if (w.level[(size_t)x] != L) continue;
      const int m = w.visit(x, L + 1);
      activated |= m > 0;
      if (last && m > 0) {
        Tail<T> g{w, L + 1};
        cp_tail_walk(g, (int32_t)x);
      }
    }
    if (!activated) break;
  }
  std::vector<double> best((size_t)n_in, -1.0);
  for (int64_t x = 0; x < N; ++x) {
    if (!on_path[x]) continue;
    const int32_t r = root[x];
    if (self_us[x] > best[(size_t)r]) {        // node order: the first node with the largest self time
      best[(size_t)r] = self_us[x];
      culprit[r] = (int32_t)x;
    }
  }
  for (int p = 0; p < P; ++p) {
    double s0 = 0.0, s1 = 0.0;
    int32_t c0 = 0, c1 = 0;
    for (int64_t x = b.prob_in_off[p]; x < b.prob_in_off[p + 1]; ++x) {
      if (!on_path[x]) continue;
      s0 = dadd(s0, self_us[x]);
      ++c0;
      if (slow[(size_t)root[x]]) {
        s1 = dadd(s1, self_us[x]);
        ++c1;
      }
    }
    server_us[2 * p] = s0;
    server_us[2 * p + 1] = s1;
    server_visits[2 * p] = c0;
    server_visits[2 * p + 1] = c1;
  }
  for (int ep = 0; ep < b.n_ep_total; ++ep) {
    double s0 = 0.0, s1 = 0.0;
    for (int64_t x = n_in + b.ep_out_off[ep]; x < n_in + b.ep_out_off[ep + 1]; ++x) {
      if (!on_path[x]) continue;
      s0 = dadd(s0, self_us[x]);
      if (slow[(size_t)root[x]]) s1 = dadd(s1, self_us[x]);
    }
    call_us[2 * ep] = s0;
    call_us[2 * ep + 1] = s1;
  }
}

// times: NULL for the int64 times of `b`, else the float64 ones (in_start, in_end, out_start, out_end).
// levels: the level launches (k_cp_level), the last walking what lies below it; 0 = until nothing is left.
extern "C" int twe_critical_paths(const tw_batch* b, const tw_times_f64* times, const int32_t* assign,
                                  const int32_t* in_caller, const int32_t* root, double slow_us, int levels,
                                  uint8_t* on_path, double* self_us, int32_t* culprit, double* server_us,
                                  int32_t* server_visits, double* call_us, int32_t* requests) {
  if (times)
    walk<double>(*b, times->in_start, times->in_end, times->out_start, times->out_end, assign, in_caller, root,
                 slow_us, levels, on_path, self_us, culprit, server_us, server_visits, call_us, requests);
  else
    walk<int64_t>(*b, b->in_start, b->in_end, b->out_start, b->out_end, assign, in_caller, root, slow_us, levels,
                  on_path, self_us, culprit, server_us, server_visits, call_us, requests);
  return TW_OK;
}
