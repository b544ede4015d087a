// tw_truth.cu — ground truth, invocation order and accuracy on the device (SURVEY.md §8 row f-2).
//
// Replaces (reference: src/trace_reconstructor/ports/python/)
//   utils.GetGroundTruth                  helpers/utils.py:22-32   O(n_in * E * n_out) list scans
//   FindOrder                             executor.py:214-285      per-trace pruning of the complete digraph
//   utils.AccuracyForService / TopKAccuracyForService / AccuracyEndToEnd / TopKAccuracyEndToEnd
//                                         helpers/utils.py:62-145
// All of them are joins on the trace id.  The loader numbers the traces densely (int32), so the joins
// are scatter / gather through a table indexed by trace number — no sort, every span read once:
// HBM-bound, 4 B per span for the truth, 4 B * E per in-span for the order and the accuracies.
#include "tw_kernels.cuh"

namespace tw {

// Table of problem p: tab[tab_off[p] + e * range_p + (trace - lo_p)] = smallest list position of a span
// of that trace in callee e's list (GetGroundTruth takes the FIRST match in list order, utils.py:28-31);
// only traces of the problem's own in-spans (lo_p <= trace < lo_p + range_p) can match.
__global__ void k_truth_scatter(tw_batch b, const int32_t* __restrict__ out_trace, const int32_t* __restrict__ trace_lo,
                                const int32_t* __restrict__ trace_n, const int64_t* __restrict__ tab_off,
                                int32_t* __restrict__ tab) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= b.n_out_total) return;
  const int ep = last_le(b.ep_out_off, b.n_ep_total, j);
  const int p = last_le(b.prob_ep_off, b.n_problems, ep);
  const int t = out_trace[j] - trace_lo[p];
  if (t >= 0 && t < trace_n[p])
    atomicMin(&tab[tab_off[p] + (int64_t)(ep - b.prob_ep_off[p]) * trace_n[p] + t], (int32_t)(j - b.ep_out_off[ep]));
}

// truth[tuple_off[p] + e * n_p + i] = table entry of the in-span's trace, or -1
__global__ void k_truth_gather(tw_batch b, const int32_t* __restrict__ in_trace, const int32_t* __restrict__ trace_lo,
                               const int32_t* __restrict__ trace_n, const int64_t* __restrict__ tab_off,
                               const int32_t* __restrict__ tab, const int32_t* __restrict__ in_prob,
                               int32_t* __restrict__ truth) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= b.n_in_total) return;
  const int p = in_prob[g];
  const int64_t in_off = b.prob_in_off[p];
  const int n = (int)(b.prob_in_off[p + 1] - in_off);
  const int i = (int)(g - in_off);
  const int E = b.prob_ep_off[p + 1] - b.prob_ep_off[p];
  const int t = in_trace[g] - trace_lo[p];
  for (int e = 0; e < E; ++e) {
    int32_t v = -1;
    if (t >= 0 && t < trace_n[p]) {
      v = tab[tab_off[p] + (int64_t)e * trace_n[p] + t];
      if (v >= 0x7f7f7f7f) v = -1;             // the fill pattern: no span of that trace
    }
    truth[b.prob_tuple_off[p] + (int64_t)e * n + i] = v;
  }
}

// FindOrder: edge a -> b of the complete digraph over a service's callees survives iff NO in-span has
// its child at a ending after its child at b starts (executor.py:248-266: x.end > y.start removes
// x.ep -> y.ep, for every ordered pair).  violated[ep0 + a] gets bit b.
__global__ void k_find_order(tw_batch b, const int32_t* __restrict__ truth, const int32_t* __restrict__ in_prob,
                             uint32_t* __restrict__ violated, int* __restrict__ missing) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= b.n_in_total) return;
  const int p = in_prob[g];
  const int64_t in_off = b.prob_in_off[p];
  const int n = (int)(b.prob_in_off[p + 1] - in_off);
  const int i = (int)(g - in_off);
  const int ep0 = b.prob_ep_off[p], E = b.prob_ep_off[p + 1] - ep0;
  int64_t s[TW_MAX_E], en[TW_MAX_E];
  for (int e = 0; e < E; ++e) {
    const int c = truth[b.prob_tuple_off[p] + (int64_t)e * n + i];
    if (c < 0) { atomicExch(missing, 1); return; }            // all_spans[...] KeyError in the reference
    const int64_t o = b.ep_out_off[ep0 + e] + c;
    s[e] = b.out_start[o];
    en[e] = b.out_end[o];
  }
  for (int a = 0; a < E; ++a) {
    uint32_t m = 0;
    for (int c = 0; c < E; ++c)
      if (c != a && en[a] > s[c]) m |= 1u << c;
    if (m & ~violated[ep0 + a]) atomicOr(&violated[ep0 + a], m);
  }
}

// Accuracies.  Per in-span: right at every callee (utils.py:62-79) / some rank right at every callee
// (:81-97).  Per trace (:99-145): `bad` / `seen` flags for AccuracyEndToEnd; TopKAccuracyEndToEnd keeps
// its order dependence — `first` marks the first service of the caller's order (there the LAST in-span
// of a trace decides: 64-bit max of (position, hit)), later services only clear the flag.
__global__ void k_accuracy(tw_batch b, const int32_t* __restrict__ truth, const int32_t* __restrict__ assign,
                           const int32_t* __restrict__ topk_idx, const uint8_t* __restrict__ topk_cnt,
                           const int32_t* __restrict__ in_trace, const int32_t* __restrict__ in_prob,
                           const uint8_t* __restrict__ prob_first, int n_traces,
                           unsigned long long* __restrict__ per_prob, uint8_t* __restrict__ trace_seen,
                           uint8_t* __restrict__ trace_bad, unsigned long long* __restrict__ trace_first,
                           uint8_t* __restrict__ trace_kbad) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= b.n_in_total) return;
  const int p = in_prob[g];
  const int64_t in_off = b.prob_in_off[p];
  const int n = (int)(b.prob_in_off[p + 1] - in_off);
  const int i = (int)(g - in_off);
  const int ep0 = b.prob_ep_off[p], E = b.prob_ep_off[p + 1] - ep0;
  const int64_t to = b.prob_tuple_off[p];
  bool ok = true;
  for (int e = 0; e < E; ++e) ok = ok && assign[to + (int64_t)e * n + i] == truth[to + (int64_t)e * n + i];
  bool hit = false;
  if (topk_idx) {
    const int cnt = topk_cnt[g];
    for (int r = 0; r < cnt && !hit; ++r) {
      bool all = true;
      for (int e = 0; e < E; ++e)
        all = all && topk_idx[TW_K * (to + (int64_t)i * E) + r * E + e] == truth[to + (int64_t)e * n + i];
      hit = all;
    }
  }
  if (ok) atomicAdd(&per_prob[2 * p], 1ull);
  if (hit) atomicAdd(&per_prob[2 * p + 1], 1ull);
  const int t = in_trace ? in_trace[g] : -1;
  if (t >= 0 && t < n_traces) {
    trace_seen[t] = 1;
    if (!ok) trace_bad[t] = 1;
    if (topk_idx) {
      if (prob_first && prob_first[p]) atomicMax(&trace_first[t], ((unsigned long long)(g + 1) << 1) | (hit ? 1ull : 0ull));
      else if (!hit) trace_kbad[t] = 1;
    }
  }
}

// traces seen / right / right within the top K: one pass over the flags
__global__ void k_accuracy_reduce(int n_traces, const uint8_t* __restrict__ seen, const uint8_t* __restrict__ bad,
                                  const unsigned long long* __restrict__ first, const uint8_t* __restrict__ kbad,
                                  unsigned long long* __restrict__ out4) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned s = 0, r = 0, ks = 0, kr = 0;
  if (t < n_traces && seen[t]) {
    s = 1;
    r = !bad[t];
    // TopKAccuracyEndToEnd: a trace absent from the first service enters with the value the first later
    // in-span gives it; `first == 0` (never set) and no later miss counts as right, like the reference's
    // `trace_acc[tid] = True` path (utils.py:131)
    ks = 1;
    const bool f = first[t] == 0ull ? true : (first[t] & 1ull) != 0;
    kr = f && !kbad[t];
  }
  const unsigned lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, d);
    r += __shfl_xor_sync(0xffffffffu, r, d);
    ks += __shfl_xor_sync(0xffffffffu, ks, d);
    kr += __shfl_xor_sync(0xffffffffu, kr, d);
  }
  if (lane == 0 && s) {
    atomicAdd(&out4[0], (unsigned long long)s);
    atomicAdd(&out4[1], (unsigned long long)r);
    atomicAdd(&out4[2], (unsigned long long)ks);
    atomicAdd(&out4[3], (unsigned long long)kr);
  }
}

__global__ void k_in_prob(tw_batch b, int32_t* __restrict__ in_prob) {
  const int p = blockIdx.x;
  const int64_t a = b.prob_in_off[p], z = b.prob_in_off[p + 1];
  for (int64_t g = a + threadIdx.x; g < z; g += blockDim.x) in_prob[g] = p;
}

cudaError_t launch_in_prob(const tw_batch& b, int32_t* in_prob, cudaStream_t s, int64_t& launches) {
  k_in_prob<<<b.n_problems, 128, 0, s>>>(b, in_prob);
  return after_launch(launches);
}

cudaError_t launch_ground_truth(const tw_batch& b, const int32_t* in_trace, const int32_t* out_trace,
                                const int32_t* trace_lo, const int32_t* trace_n, const int64_t* tab_off, int64_t tab_len,
                                int32_t* tab, const int32_t* in_prob, int32_t* truth, cudaStream_t s,
                                int64_t& launches) {
  cudaError_t e = cudaMemsetAsync(tab, 0x7f, (size_t)tab_len * sizeof(int32_t), s);   // "no position yet"
  if (e != cudaSuccess) return e;
  if (b.n_out_total > 0) {
    k_truth_scatter<<<(unsigned)((b.n_out_total + 255) / 256), 256, 0, s>>>(b, out_trace, trace_lo, trace_n, tab_off, tab);
    e = after_launch(launches);
    if (e != cudaSuccess) return e;
  }
  k_truth_gather<<<(unsigned)((b.n_in_total + 255) / 256), 256, 0, s>>>(b, in_trace, trace_lo, trace_n, tab_off, tab, in_prob,
                                                                        truth);
  return after_launch(launches);
}

cudaError_t launch_find_order(const tw_batch& b, const int32_t* truth, const int32_t* in_prob, uint32_t* violated,
                              int* missing, cudaStream_t s, int64_t& launches) {
  cudaError_t e = cudaMemsetAsync(violated, 0, (size_t)b.n_ep_total * sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  e = cudaMemsetAsync(missing, 0, sizeof(int), s);
  if (e != cudaSuccess) return e;
  k_find_order<<<(unsigned)((b.n_in_total + 255) / 256), 256, 0, s>>>(b, truth, in_prob, violated, missing);
  return after_launch(launches);
}

cudaError_t launch_accuracy(const tw_batch& b, const int32_t* truth, const int32_t* assign, const int32_t* topk_idx,
                            const uint8_t* topk_cnt, const int32_t* in_trace, const int32_t* in_prob,
                            const uint8_t* prob_first, int n_traces, unsigned long long* per_prob, uint8_t* flags,
                            unsigned long long* trace_first, unsigned long long* out4, cudaStream_t s,
                            int64_t& launches) {
  uint8_t* seen = flags;
  uint8_t* bad = flags + n_traces;
  uint8_t* kbad = flags + 2 * (size_t)n_traces;
  k_accuracy<<<(unsigned)((b.n_in_total + 255) / 256), 256, 0, s>>>(b, truth, assign, topk_idx, topk_cnt, in_trace, in_prob,
                                                                    prob_first, n_traces, per_prob, seen, bad, trace_first,
                                                                    kbad);
  cudaError_t e = after_launch(launches);
  if (e != cudaSuccess || n_traces == 0) return e;
  k_accuracy_reduce<<<(n_traces + 255) / 256, 256, 0, s>>>(n_traces, seen, bad, trace_first, kbad, out4);
  return after_launch(launches);
}

}  // namespace tw
