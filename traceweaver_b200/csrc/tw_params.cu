// tw_params.cu — order-statistics delay parameters of pass 0, and the delay samples fed to the
// pass-boundary refit.
//
// Replaces (V3 = traceweaver_v3.py)
//   ComputeEpPairDistParams3           V3:580-646   (sorted arrival/departure arrays, 100-span
//                                                    slices, mean + batch-means std via tstd)
//   `durations` of ComputeEpPairDistParams5  V3:721-760
#include "tw_kernels.cuh"

namespace tw {

// ---------------------------------------------------------------------------------------------
// Segmented sort of the END timestamps (starts arrive sorted, ends do not): one CTA per segment,
// bitonic network in shared memory.  Segments: P in-span lists, then n_ep_total out-span lists.
// ---------------------------------------------------------------------------------------------
constexpr int kSortThreads = 256;

__global__ void __launch_bounds__(kSortThreads)
k_sort_ends(tw_batch b, int64_t* __restrict__ in_end_sorted, int64_t* __restrict__ out_end_sorted,
            int pow2_cap, int* __restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int64_t* a = reinterpret_cast<int64_t*>(smem_raw);
  const int seg = blockIdx.x;
  const int64_t* src;
  int64_t* dst;
  int n;
  if (seg < b.n_problems) {
    int64_t off = b.prob_in_off[seg];
    n = (int)(b.prob_in_off[seg + 1] - off);
    src = b.in_end + off;
    dst = in_end_sorted + off;
  } else {
    int ep = seg - b.n_problems;
    int64_t off = b.ep_out_off[ep];
    n = (int)(b.ep_out_off[ep + 1] - off);
    src = b.out_end + off;
    dst = out_end_sorted + off;
  }
  if (n > pow2_cap) return;      // long lists are sorted in global memory by k_sort_ends_long
  int m = 1;
  while (m < n) m <<= 1;
  for (int x = threadIdx.x; x < m; x += kSortThreads) a[x] = x < n ? src[x] : INT64_MAX;
  __syncthreads();
  for (int k = 2; k <= m; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int x = threadIdx.x; x < m; x += kSortThreads) {
        int y = x ^ j;
        if (y > x) {
          bool up = (x & k) == 0;
          int64_t ax = a[x], ay = a[y];
          if ((ax > ay) == up) { a[x] = ay; a[y] = ax; }
        }
      }
      __syncthreads();
    }
  }
  for (int x = threadIdx.x; x < n; x += kSortThreads) dst[x] = a[x];
}

// Lists longer than the shared-memory network (one service with tens of thousands of spans): the same
// bitonic network on a power-of-two scratch slab in global memory, one 1024-thread CTA per list.
// long_seg[k] = segment id as above; slab k starts at scratch + k * slab_len.
__global__ void __launch_bounds__(1024)
k_sort_ends_long(tw_batch b, const int32_t* __restrict__ long_seg, int64_t* __restrict__ scratch, int64_t slab_len,
                 int64_t* __restrict__ in_end_sorted, int64_t* __restrict__ out_end_sorted) {
  const int seg = long_seg[blockIdx.x];
  int64_t* a = scratch + (int64_t)blockIdx.x * slab_len;
  const int64_t* src;
  int64_t* dst;
  int n;
  if (seg < b.n_problems) {
    int64_t off = b.prob_in_off[seg];
    n = (int)(b.prob_in_off[seg + 1] - off);
    src = b.in_end + off;
    dst = in_end_sorted + off;
  } else {
    int ep = seg - b.n_problems;
    int64_t off = b.ep_out_off[ep];
    n = (int)(b.ep_out_off[ep + 1] - off);
    src = b.out_end + off;
    dst = out_end_sorted + off;
  }
  int m = 1;
  while (m < n) m <<= 1;
  for (int x = threadIdx.x; x < m; x += blockDim.x) a[x] = x < n ? src[x] : INT64_MAX;
  __syncthreads();
  for (int k = 2; k <= m; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int x = threadIdx.x; x < m; x += blockDim.x) {
        int y = x ^ j;
        if (y > x) {
          bool up = (x & k) == 0;
          int64_t ax = a[x], ay = a[y];
          if ((ax > ay) == up) { a[x] = ay; a[y] = ax; }
        }
      }
      __syncthreads();
    }
  }
  for (int x = threadIdx.x; x < n; x += blockDim.x) dst[x] = a[x];
}

cudaError_t setup_sort_ends() {
  return cudaFuncSetAttribute(k_sort_ends, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)(kSortSmemCap * sizeof(int64_t)));
}

cudaError_t launch_sort_ends(const tw_batch& b, int64_t* in_end_sorted, int64_t* out_end_sorted,
                             int max_seg, const int32_t* long_seg, int n_long, int64_t* long_scratch,
                             int64_t slab_len, int* err_flag, cudaStream_t s, int64_t& launches) {
  int cap = 1;
  while (cap < max_seg && cap < kSortSmemCap) cap <<= 1;
  size_t smem = (size_t)cap * sizeof(int64_t);
  k_sort_ends<<<b.n_problems + b.n_ep_total, kSortThreads, smem, s>>>(b, in_end_sorted, out_end_sorted, cap,
                                                                       err_flag);
  cudaError_t e = after_launch(launches);
  if (e != cudaSuccess) return e;
  if (n_long > 0) {
    k_sort_ends_long<<<n_long, 1024, 0, s>>>(b, long_seg, long_scratch, slab_len, in_end_sorted, out_end_sorted);
    e = after_launch(launches);
  }
  return e;
}

// ---------------------------------------------------------------------------------------------
// ComputeDistParams, V3:590-617.  One warp per (problem, 100-span batch); integer sums are exact
// so the lane-parallel reduction reproduces Python's int arithmetic; the float tail runs on lane
// 0 with numpy's summation order (pairwise, 8 lanes) and scipy's tstd formula.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double np_sum10(const double* a, int n) {
  if (n < 8) {
    double r = 0.0;
    for (int i = 0; i < n; ++i) r = dadd(r, a[i]);
    return r;
  }
  double r[8];
  for (int j = 0; j < 8; ++j) r[j] = a[j];
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] = dadd(r[j], a[i + j]);
  double res = dadd(dadd(dadd(r[0], r[1]), dadd(r[2], r[3])), dadd(dadd(r[4], r[5]), dadd(r[6], r[7])));
  for (; i < n; ++i) res = dadd(res, a[i]);
  return res;
}

__device__ __forceinline__ double tstd_dev(const double* x, int n) {
  double mean = ddiv(np_sum10(x, n), (double)n);
  double d[TW_PARAM_NBATCHES];
  for (int i = 0; i < n; ++i) { double t = dsub(x[i], mean); d[i] = dmul(t, t); }
  double var = ddiv(np_sum10(d, n), (double)n);
  if (n - 1 <= 0) return __longlong_as_double(0x7ff8000000000000LL);
  var = dmul(var, ddiv((double)n, (double)(n - 1)));
  return sqrt(var);
}

// kShifted: the batch's timestamps are fixed-point values x * 2^prob_shift[p] (tw_engine_bind_f64).  The bin
// sums stay exact integers; the total and the batch means are taken back to real microseconds (ldexp is
// exact) before the float tail, so the records, the sigma clamp and log(sigma) are in real units.
template <bool kShifted>
__global__ void __launch_bounds__(128)
k_params0(tw_batch b, const int64_t* __restrict__ in_end_sorted, const int64_t* __restrict__ out_end_sorted,
          const int64_t* __restrict__ prob_gauss_off, const int32_t* __restrict__ batch_prob,
          const int32_t* __restrict__ batch_idx, int n_batches_total, double* __restrict__ gauss_out,
          const int32_t* __restrict__ prob_shift) {
  const int wid = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (wid >= n_batches_total) return;
  const int p = batch_prob[wid], bt = batch_idx[wid];
  const int64_t in_off = b.prob_in_off[p];
  const int n = (int)(b.prob_in_off[p + 1] - in_off);
  const int ep0 = b.prob_ep_off[p], E = b.prob_ep_off[p + 1] - ep0;
  const int term0 = b.ep_term_off[ep0];
  const int n_terms = b.ep_term_off[ep0 + E] - term0;
  const int s = bt * TW_PARAM_BATCH;
  const int z = min(n, s + TW_PARAM_BATCH);
  const int m = z - s;
  const int bs = (m + TW_PARAM_NBATCHES - 1) / TW_PARAM_NBATCHES;
  for (int e = 0; e < E; ++e) {
    const int64_t oo = b.ep_out_off[ep0 + e];
    for (int t = b.ep_term_off[ep0 + e] - term0; t < b.ep_term_off[ep0 + e + 1] - term0; ++t) {
      const int src = b.term_src[term0 + t];
      const int64_t *t1, *t2;
      if (src >= 0) { t1 = out_end_sorted + b.ep_out_off[ep0 + src]; t2 = b.out_start + oo; }     // V3:640-642
      else if (src == TW_TERM_ROOT) { t1 = b.in_start + in_off; t2 = b.out_start + oo; }          // V3:623-626
      else { t1 = out_end_sorted + oo; t2 = in_end_sorted + in_off; }                             // V3:644-646
      long long bin[TW_PARAM_NBATCHES];
#pragma unroll
      for (int q = 0; q < TW_PARAM_NBATCHES; ++q) bin[q] = 0;
      for (int j = s + lane; j < z; j += 32) {
        long long d = t2[j] - t1[j];
        int q = (j - s) / bs;
#pragma unroll
        for (int qq = 0; qq < TW_PARAM_NBATCHES; ++qq)
          if (qq == q) bin[qq] += d;
      }
#pragma unroll
      for (int q = 0; q < TW_PARAM_NBATCHES; ++q)
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) bin[q] += __shfl_xor_sync(0xffffffffu, bin[q], d);
      if (lane == 0) {
        long long tot = 0;
        double bm[TW_PARAM_NBATCHES];
        int nb = 0;
#pragma unroll
        for (int q = 0; q < TW_PARAM_NBATCHES; ++q) {
          tot += bin[q];
          int a0 = q * bs, z0 = min(m, (q + 1) * bs);
          if (z0 - a0 > 0) {
            if constexpr (kShifted) bm[nb++] = ddiv(ldexp((double)bin[q], -prob_shift[p]), (double)(z0 - a0));
            else bm[nb++] = ddiv((double)bin[q], (double)(z0 - a0));
          }
        }
        double mean;
        if constexpr (kShifted) mean = ddiv(ldexp((double)tot, -prob_shift[p]), (double)m);
        else mean = ddiv((double)tot, (double)m);
        double sd = dmul(sqrt((double)bs), tstd_dev(bm, nb));
        if (sd < 1.0e-12) sd = 0.001;                                   // V1:130-131
        double* rec = gauss_out + (prob_gauss_off[p] + (int64_t)bt * n_terms + t) * TW_GAUSS_REC;
        rec[0] = mean; rec[1] = sd; rec[2] = log(sd);
      }
    }
  }
}

cudaError_t launch_params0(const tw_batch& b, const int64_t* in_end_sorted, const int64_t* out_end_sorted,
                           const int64_t* prob_gauss_off, const int32_t* batch_prob, const int32_t* batch_idx,
                           int n_batches_total, double* gauss_out, const int32_t* prob_shift, cudaStream_t s,
                           int64_t& launches) {
  int blocks = (n_batches_total + 3) / 4;
  if (prob_shift)
    k_params0<true><<<blocks, 128, 0, s>>>(b, in_end_sorted, out_end_sorted, prob_gauss_off, batch_prob, batch_idx,
                                           n_batches_total, gauss_out, prob_shift);
  else
    k_params0<false><<<blocks, 128, 0, s>>>(b, in_end_sorted, out_end_sorted, prob_gauss_off, batch_prob, batch_idx,
                                            n_batches_total, gauss_out, nullptr);
  return after_launch(launches);
}

// ---------------------------------------------------------------------------------------------
// Delay samples per term from a pass's assignments (V3:721-760).  One warp per term, ballot
// compaction keeps in-span order (the refit's k-means++ seeding indexes samples by position).
// ---------------------------------------------------------------------------------------------
// kShifted: fixed-point timestamps (see k_params0); the exact integer difference is converted, then scaled
// back to real microseconds by ldexp, which is exact.
template <bool kShifted>
__global__ void __launch_bounds__(128)
k_delays(tw_batch b, const int32_t* __restrict__ assign, const int64_t* __restrict__ term_sample_off,
         const int32_t* __restrict__ term_ep, const int32_t* __restrict__ ep_prob,
         double* __restrict__ delays, int32_t* __restrict__ counts, const int32_t* __restrict__ prob_shift) {
  const int t = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= b.n_term_total) return;
  const int ep = term_ep[t];
  const int p = ep_prob[ep];
  const int ep0 = b.prob_ep_off[p];
  const int e = ep - ep0;
  const int64_t in_off = b.prob_in_off[p];
  const int n = (int)(b.prob_in_off[p + 1] - in_off);
  const int64_t tuple_off = b.prob_tuple_off[p];
  const int src = b.term_src[t];
  const int64_t* os_e = b.out_start + b.ep_out_off[ep];
  const int64_t* oe_e = b.out_end + b.ep_out_off[ep];
  const int64_t* oe_b = src >= 0 ? b.out_end + b.ep_out_off[ep0 + src] : nullptr;
  const int32_t* a_e = assign + tuple_off + (int64_t)e * n;
  const int32_t* a_b = src >= 0 ? assign + tuple_off + (int64_t)src * n : nullptr;
  double* dst = delays + term_sample_off[t];
  int base = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    int i = i0 + lane;
    bool ok = false;
    double d = 0.0;
    if (i < n) {
      int ce = a_e[i];
      if (ce >= 0) {
        if (src >= 0) {
          int cb = a_b[i];
          if (cb >= 0) { ok = true; d = (double)(os_e[ce] - oe_b[cb]); }
        } else if (src == TW_TERM_ROOT) { ok = true; d = (double)(os_e[ce] - b.in_start[in_off + i]); }
        else { ok = true; d = (double)(b.in_end[in_off + i] - oe_e[ce]); }
      }
    }
    if constexpr (kShifted) d = ldexp(d, -prob_shift[p]);
    unsigned mask = __ballot_sync(0xffffffffu, ok);
    if (ok) dst[base + __popc(mask & ((1u << lane) - 1u))] = d;
    base += __popc(mask);
  }
  if (lane == 0) counts[t] = base;
}

cudaError_t launch_delays(const tw_batch& b, const int32_t* assign, const int64_t* term_sample_off,
                          const int32_t* term_ep, const int32_t* ep_prob, double* delays, int32_t* counts,
                          const int32_t* prob_shift, cudaStream_t s, int64_t& launches) {
  int blocks = (b.n_term_total + 3) / 4;
  if (prob_shift)
    k_delays<true><<<blocks, 128, 0, s>>>(b, assign, term_sample_off, term_ep, ep_prob, delays, counts, prob_shift);
  else
    k_delays<false><<<blocks, 128, 0, s>>>(b, assign, term_sample_off, term_ep, ep_prob, delays, counts, nullptr);
  return after_launch(launches);
}

}  // namespace tw
