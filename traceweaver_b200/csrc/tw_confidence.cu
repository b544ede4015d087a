// tw_confidence.cu — confidence of the reconstructed requests (tw_request_confidence).
//
// After the join (tw_traces.cu) every in-span is one reconstruction decision of a request.  One thread per
// in-span reads its chosen tuple, score and code and its final top-K row, forms its choice probability p and
// -log p in fixed point (conf_choice, tw_core.cuh) and scatters them into its root's counters with integer
// atomics.  Then every request's confidence and weakest decision (an integer min over the bits of the
// non-negative p, then a min over the node ids that hold it), and the per-service means and batch total, one
// CTA per service in a fixed order.  No float atomics: every result is the same from run to run, for any grid.
#include "tw_kernels.cuh"

namespace tw {

namespace {

// One thread per in-span x: p and ell, and into the counters of its root r (an in-span root: x belongs to a
// request) the decision, a zero or the fixed-point ell, and the smallest p bits.  Also sets weakest[x] to
// INT_MAX for a root and -1 otherwise.
__global__ void __launch_bounds__(kTreeThreads)
k_conf_step(tw_batch bt, const int32_t* __restrict__ assign, const double* __restrict__ score,
            const uint8_t* __restrict__ code, tw_score_out top, tw_confidence_out out,
            unsigned long long* __restrict__ wbits) {
  const int64_t n_in = bt.n_in_total;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_in; g += (int64_t)gridDim.x * blockDim.x) {
    const int p = last_le(bt.prob_in_off, bt.n_problems, g);
    const int64_t in0 = bt.prob_in_off[p], n = bt.prob_in_off[p + 1] - in0, i = g - in0;
    const int E = bt.prob_ep_off[p + 1] - bt.prob_ep_off[p];
    const int64_t tup = bt.prob_tuple_off[p];
    int32_t c[TW_MAX_E];
    for (int e = 0; e < E; ++e) c[e] = assign[tup + e * n + i];
    const ConfChoice ch = conf_choice(E, c, code[g], score[g], top.topk_score + g * TW_K,
                                      top.topk_idx + TW_K * (tup + i * E), top.topk_cnt[g]);
    out.p[g] = ch.p;
    out.ell[g] = ch.ell;
    const int32_t r = out.root[g];
    out.weakest[g] = r == (int32_t)g ? 0x7fffffff : -1;
    if (r < 0 || r >= n_in) continue;                   // on or under a cycle, or a detached fragment
    atomicAdd(&out.decisions[r], 1);
    if (ch.q < 0) atomicAdd(&out.zero[r], 1);
    else atomicAdd((unsigned long long*)&out.log_conf[r], (unsigned long long)ch.q);
    atomicMin(&wbits[r], (unsigned long long)conf_bits(ch.p));
  }
}

// One thread per in-span: the weakest decision of its request (smallest node id whose p bits are the
// request's minimum); for a root its confidence, weakest p and the size check (flag: the smallest root with
// TW_CONF_MAX_DECISIONS or more decisions).  NaN conf / weakest_p for any other in-span.
__global__ void __launch_bounds__(kTreeThreads)
k_conf_root(int64_t n_in, tw_confidence_out out, const unsigned long long* __restrict__ wbits,
            int32_t* __restrict__ flag) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_in; g += (int64_t)gridDim.x * blockDim.x) {
    const int32_t r = out.root[g];
    if (r >= 0 && r < n_in && conf_bits(out.p[g]) == wbits[r]) atomicMin(&out.weakest[r], (int32_t)g);
    if (r != (int32_t)g) {
      out.conf[g] = tw_nan();
      out.weakest_p[g] = tw_nan();
      continue;
    }
    out.conf[g] = conf_request(out.log_conf[g], out.zero[g]);
    out.weakest_p[g] = conf_from_bits(wbits[g]);
    if (out.decisions[g] >= TW_CONF_MAX_DECISIONS) atomicMin(flag, (int32_t)g);
  }
}

// One CTA per service: est_accuracy (the mean p of its in-spans), and the sum of conf over the request
// roots among them with their count (seg_conf / seg_req, for k_conf_total).
__global__ void __launch_bounds__(kTreeThreads)
k_conf_reduce(tw_batch bt, tw_confidence_out out, double* __restrict__ seg_conf, int32_t* __restrict__ seg_req) {
  __shared__ double ws[1][kTreeThreads / 32];
  __shared__ int wc[1][kTreeThreads / 32];
  for (int sg = blockIdx.x; sg < bt.n_problems; sg += gridDim.x) {
    const int64_t lo = bt.prob_in_off[sg], hi = bt.prob_in_off[sg + 1];
    double s[1];
    int c[1];
    tree_cta_sum(lo, hi, [&](int64_t x, double* a, int*) { a[0] = dadd(a[0], out.p[x]); }, ws, wc, s, c);
    if (threadIdx.x == 0) out.est_accuracy[sg] = ddiv(s[0], (double)(hi - lo));
    tree_cta_sum(lo, hi, [&](int64_t x, double* a, int* k) {
      if (out.root[x] == (int32_t)x) {
        a[0] = dadd(a[0], out.conf[x]);
        ++k[0];
      }
    }, ws, wc, s, c);
    if (threadIdx.x == 0) {
      seg_conf[sg] = s[0];
      seg_req[sg] = c[0];
    }
  }
}

// One CTA: the batch's request count and expected_exact from the services' partials, in the same order.
__global__ void __launch_bounds__(kTreeThreads)
k_conf_total(int n_problems, const double* __restrict__ seg_conf, const int32_t* __restrict__ seg_req,
             tw_confidence_out out) {
  __shared__ double ws[1][kTreeThreads / 32];
  __shared__ int wc[1][kTreeThreads / 32];
  double s[1];
  int c[1];
  tree_cta_sum(0, n_problems, [&](int64_t x, double* a, int* k) {
    a[0] = dadd(a[0], seg_conf[x]);
    k[0] += seg_req[x];
  }, ws, wc, s, c);
  if (threadIdx.x == 0) {
    out.expected_exact[0] = s[0];
    out.requests[0] = c[0];
  }
}

}  // namespace

cudaError_t launch_request_confidence(const tw_batch& b, const int32_t* assign, const double* score,
                                      const uint8_t* code, const tw_score_out& top, const tw_confidence_out& out,
                                      const CfScratch& sc, int n_sm, cudaStream_t s, int64_t& launches) {
  const int64_t n_in = b.n_in_total;
  cudaError_t e;
  if ((e = cudaMemsetAsync(out.decisions, 0, (size_t)n_in * sizeof(int32_t), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(out.zero, 0, (size_t)n_in * sizeof(int32_t), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(out.log_conf, 0, (size_t)n_in * sizeof(int64_t), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(sc.wbits, 0xff, (size_t)n_in * sizeof(unsigned long long), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(sc.flag, 0x7f, sizeof(int32_t), s)) != cudaSuccess) return e;
  const unsigned g = tree_grid(n_in, n_sm);
  k_conf_step<<<g, kTreeThreads, 0, s>>>(b, assign, score, code, top, out, sc.wbits);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  k_conf_root<<<g, kTreeThreads, 0, s>>>(n_in, out, sc.wbits, sc.flag);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  const int64_t cap = (int64_t)n_sm * 8;
  k_conf_reduce<<<(unsigned)(b.n_problems < cap ? b.n_problems : cap), kTreeThreads, 0, s>>>(b, out, sc.seg_conf,
                                                                                           sc.seg_req);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  k_conf_total<<<1, kTreeThreads, 0, s>>>(b.n_problems, sc.seg_conf, sc.seg_req, out);
  return after_launch(launches);
}

}  // namespace tw
