// tw_times.cu — float64 microsecond timestamps: the spans executor.py --compress_factor > 1 produces
// (transforms.repeat_change_spans divides start times by the factor).
//
// Every problem p is moved into exact fixed point: s_p = the smallest shift such that x * 2^s_p is an
// integer for every start and end time of p, X = x * 2^s_p in int64.  The map is monotone and exact, so
// every comparison of the engine gives the same answer on X as on x; (double)(X_a - X_b) equals
// round(x_a - x_b) * 2^s_p; the scoring kernels run unchanged on X with rescaled parameter records
// (k_params_scale), and pass 0 / the delays are taken back to real microseconds (tw_params.cu).
#include "tw_kernels.cuh"

namespace tw {

constexpr int kTimesThreads = 256;

// Problem of element j of [in-spans | out-spans]: offsets are strictly increasing (n_in >= 2, n_out >= 1).
__device__ __forceinline__ int elem_problem(const tw_batch& b, const int32_t* __restrict__ ep_prob, int64_t j) {
  const int64_t* off = b.prob_in_off;
  int n = b.n_problems;
  if (j >= b.n_in_total) { j -= b.n_in_total; off = b.ep_out_off; n = b.n_ep_total; }
  const int k = last_le(off, n, j);
  return off == b.prob_in_off ? k : ep_prob[k];
}

// Bits after the binary point of x (0 for integers and zero) and floor(log2 |x|) (very negative for
// zero); kShiftInvalid for NaN / inf.
__device__ __forceinline__ void time_bits(double x, int& frac, int& top) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(x);
  const int ef = (int)((u >> 52) & 0x7ff);
  unsigned long long m = u & ((1ull << 52) - 1);
  if (ef == 0x7ff) { frac = kShiftInvalid; top = 0; return; }
  if (ef == 0 && m == 0) { frac = 0; top = -4096; return; }
  if (ef != 0) m |= 1ull << 52;
  const int e = (ef ? ef : 1) - 1023 - 52;                  // x = m * 2^e
  const int f = -e - (__ffsll((long long)m) - 1);
  frac = f > 0 ? f : 0;
  top = e + 63 - __clzll((long long)m);
}

// s_p = max over the problem's start / end times of their fractional bits; prob_top[p] = floor(log2 max|x|).
// Lanes of a warp that fall in the same problem combine before the atomics.
__global__ void __launch_bounds__(kTimesThreads)
k_time_shift(tw_batch b, TimesF64 t, const int32_t* __restrict__ ep_prob, int32_t* __restrict__ prob_shift,
             int32_t* __restrict__ prob_top) {
  const int64_t n = b.n_in_total + b.n_out_total;
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
    const int64_t j = base + lane;
    int p = -1, f = 0, top = -4096;
    if (j < n) {
      p = elem_problem(b, ep_prob, j);
      const double xs = j < b.n_in_total ? t.in_start[j] : t.out_start[j - b.n_in_total];
      const double xe = j < b.n_in_total ? t.in_end[j] : t.out_end[j - b.n_in_total];
      int f2, t2;
      time_bits(xs, f, top);
      time_bits(xe, f2, t2);
      f = max(f, f2);
      top = max(top, t2);
    }
    const unsigned grp = __match_any_sync(0xffffffffu, p);
    f = __reduce_max_sync(grp, f);
    top = __reduce_max_sync(grp, top);
    if (p >= 0 && lane == __ffs(grp) - 1) {
      if (f > 0) atomicMax(&prob_shift[p], f);
      atomicMax(&prob_top[p], top);
    }
  }
}

// X = x * 2^s_p (exact: x * 2^s_p is an integer below 2^55 in magnitude); problems that fail the
// conditions get zeros and their status.
__global__ void __launch_bounds__(kTimesThreads)
k_to_fixed(tw_batch b, TimesF64 t, const int32_t* __restrict__ ep_prob, const int32_t* __restrict__ prob_shift,
           const int32_t* __restrict__ prob_top, int64_t* __restrict__ fx, int32_t* __restrict__ prob_status) {
  const int64_t n = b.n_in_total + b.n_out_total;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const int p = elem_problem(b, ep_prob, j);
    const int s = prob_shift[p];
    const int status = s >= kShiftInvalid ? TW_ERR_INVALID
                       : prob_top[p] + s >= kFixedBits ? TW_ERR_RANGE_LIMIT : TW_OK;
    const bool in = j < b.n_in_total;
    const int64_t k = in ? j : j - b.n_in_total;
    const double xs = in ? t.in_start[k] : t.out_start[k];
    const double xe = in ? t.in_end[k] : t.out_end[k];
    int64_t* ds = in ? fx : fx + 2 * b.n_in_total;
    const int64_t len = in ? b.n_in_total : b.n_out_total;
    ds[k] = status == TW_OK ? __double2ll_rn(ldexp(xs, s)) : 0;
    ds[len + k] = status == TW_OK ? __double2ll_rn(ldexp(xe, s)) : 0;
    if (in && j == b.prob_in_off[p]) prob_status[p] = status;
  }
}

cudaError_t launch_to_fixed(const tw_batch& b, const TimesF64& t, const int32_t* ep_prob, int32_t* prob_shift,
                            int32_t* prob_top, int64_t* fx, int32_t* prob_status, cudaStream_t s, int64_t& launches) {
  const int64_t n = b.n_in_total + b.n_out_total;
  const int64_t want = (n + kTimesThreads - 1) / kTimesThreads;
  const int blocks = (int)(want < 65535 ? want : 65535);
  k_time_shift<<<blocks, kTimesThreads, 0, s>>>(b, t, ep_prob, prob_shift, prob_top);
  cudaError_t e = after_launch(launches);
  if (e != cudaSuccess) return e;
  k_to_fixed<<<blocks, kTimesThreads, 0, s>>>(b, t, ep_prob, prob_shift, prob_top, fx, prob_status);
  return after_launch(launches);
}

// Scoring copies of real-unit records for a shifted batch: dt reaches the score as (real dt) * 2^s.
//   Gaussian {mu, sigma, log sigma} -> {mu 2^s, sigma 2^s, log sigma}: (dt - mu) / sigma is bit-identical.
//   Mixture {k, pc, mu pc, log pc, log w} -> pc 2^-s: dt pc - mu pc is bit-identical; k = 0 records hold
//   a Gaussian record at rec + 1.
__global__ void __launch_bounds__(kTimesThreads)
k_params_scale(int mode, const int64_t* __restrict__ prob_gauss_off, int n_problems, const double* __restrict__ src,
               double* __restrict__ dst, int64_t n_rec, const int32_t* __restrict__ term_ep,
               const int32_t* __restrict__ ep_prob, const int32_t* __restrict__ prob_shift) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rec) return;
  if (mode == TW_PARAMS_GAUSS_BATCHED) {
    const int s = prob_shift[last_le(prob_gauss_off, n_problems, r)];
    const double* a = src + r * TW_GAUSS_REC;
    double* d = dst + r * TW_GAUSS_REC;
    d[0] = ldexp(a[0], s);
    d[1] = ldexp(a[1], s);
    d[2] = a[2];
    return;
  }
  const int s = prob_shift[ep_prob[term_ep[r]]];
  const double* a = src + r * TW_MIX_REC;
  double* d = dst + r * TW_MIX_REC;
  for (int x = 0; x < TW_MIX_REC; ++x) d[x] = a[x];
  if ((int)a[0] == 0) {
    d[1] = ldexp(a[1], s);
    d[2] = ldexp(a[2], s);
  } else {
    for (int c = 0; c < TW_GMM_MAX_COMP; ++c) d[1 + c] = ldexp(a[1 + c], -s);
  }
}

cudaError_t launch_params_scale(int mode, const int64_t* prob_gauss_off, int n_problems, const double* src,
                                double* dst, int64_t n_rec, const int32_t* term_ep, const int32_t* ep_prob,
                                const int32_t* prob_shift, cudaStream_t s, int64_t& launches) {
  if (n_rec == 0) return cudaSuccess;
  k_params_scale<<<(unsigned)((n_rec + kTimesThreads - 1) / kTimesThreads), kTimesThreads, 0, s>>>(
      mode, prob_gauss_off, n_problems, src, dst, n_rec, term_ep, ep_prob, prob_shift);
  return after_launch(launches);
}

}  // namespace tw
