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

constexpr int kCfThreads = 256;

__device__ __forceinline__ int cf_last_le(const int64_t* off, int n, int64_t key) {   // last idx with off[idx] <= key
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= key) lo = mid; else hi = mid;
  }
  return lo;
}

// One thread per in-span x: p and ell, and into the counters of its root r (an in-span root: x belongs to a
// request) the decision, a zero or the fixed-point ell, and the smallest p bits.  Also sets weakest[x] to
// INT_MAX for a root and -1 otherwise.
__global__ void __launch_bounds__(kCfThreads)
k_conf_step(tw_batch bt, const int32_t* __restrict__ assign, const double* __restrict__ score,
            const uint8_t* __restrict__ code, tw_score_out top, tw_confidence_out out,
            unsigned long long* __restrict__ wbits) {
  const int64_t n_in = bt.n_in_total;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_in; g += (int64_t)gridDim.x * blockDim.x) {
    const int p = cf_last_le(bt.prob_in_off, bt.n_problems, g);
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
__global__ void __launch_bounds__(kCfThreads)
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

// The CTA's fixed-order sum of v over [lo, hi): thread t adds the elements t, t + 256, ... in order, then a
// butterfly per warp and the warps in order.  Thread 0 gets the sum.  c counts alongside.
template <class F>
__device__ void cf_cta_sum(int64_t lo, int64_t hi, F v, double* ws, int* wc, double& s, int& c) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  s = 0.0;
  c = 0;
  for (int64_t x = lo + threadIdx.x; x < hi; x += blockDim.x) v(x, s, c);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    s = dadd(s, __shfl_xor_sync(0xffffffffu, s, d));
    c += __shfl_xor_sync(0xffffffffu, c, d);
  }
  if (lane == 0) {
    ws[warp] = s;
    wc[warp] = c;
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < kCfThreads / 32; ++w) {
      s = dadd(s, ws[w]);
      c += wc[w];
    }
  __syncthreads();
}

// One CTA per service: est_accuracy (the mean p of its in-spans), and the sum of conf over the request
// roots among them with their count (seg_conf / seg_req, for k_conf_total).
__global__ void __launch_bounds__(kCfThreads)
k_conf_reduce(tw_batch bt, tw_confidence_out out, double* __restrict__ seg_conf, int32_t* __restrict__ seg_req) {
  __shared__ double ws[kCfThreads / 32];
  __shared__ int wc[kCfThreads / 32];
  for (int sg = blockIdx.x; sg < bt.n_problems; sg += gridDim.x) {
    const int64_t lo = bt.prob_in_off[sg], hi = bt.prob_in_off[sg + 1];
    double s;
    int c;
    cf_cta_sum(lo, hi, [&](int64_t x, double& a, int&) { a = dadd(a, out.p[x]); }, ws, wc, s, c);
    if (threadIdx.x == 0) out.est_accuracy[sg] = ddiv(s, (double)(hi - lo));
    cf_cta_sum(lo, hi, [&](int64_t x, double& a, int& k) {
      if (out.root[x] == (int32_t)x) {
        a = dadd(a, out.conf[x]);
        ++k;
      }
    }, ws, wc, s, c);
    if (threadIdx.x == 0) {
      seg_conf[sg] = s;
      seg_req[sg] = c;
    }
  }
}

// One CTA: the batch's request count and expected_exact from the services' partials, in the same order.
__global__ void __launch_bounds__(kCfThreads)
k_conf_total(int n_problems, const double* __restrict__ seg_conf, const int32_t* __restrict__ seg_req,
             tw_confidence_out out) {
  __shared__ double ws[kCfThreads / 32];
  __shared__ int wc[kCfThreads / 32];
  double s;
  int c;
  cf_cta_sum(0, n_problems, [&](int64_t x, double& a, int& k) {
    a = dadd(a, seg_conf[x]);
    k += seg_req[x];
  }, ws, wc, s, c);
  if (threadIdx.x == 0) {
    out.expected_exact[0] = s;
    out.requests[0] = c;
  }
}

unsigned cf_grid(int64_t n, int n_sm) {
  const int64_t want = (n + kCfThreads - 1) / kCfThreads;
  const int64_t cap = (int64_t)n_sm * 16;
  return (unsigned)(want < 1 ? 1 : (want < cap ? want : cap));
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
  const unsigned g = cf_grid(n_in, n_sm);
  k_conf_step<<<g, kCfThreads, 0, s>>>(b, assign, score, code, top, out, sc.wbits);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  k_conf_root<<<g, kCfThreads, 0, s>>>(n_in, out, sc.wbits, sc.flag);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  const int64_t cap = (int64_t)n_sm * 8;
  k_conf_reduce<<<(unsigned)(b.n_problems < cap ? b.n_problems : cap), kCfThreads, 0, s>>>(b, out, sc.seg_conf,
                                                                                           sc.seg_req);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  k_conf_total<<<1, kCfThreads, 0, s>>>(b.n_problems, sc.seg_conf, sc.seg_req, out);
  return after_launch(launches);
}

}  // namespace tw
