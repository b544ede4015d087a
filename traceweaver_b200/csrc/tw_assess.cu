// tw_assess.cu — tw_score_assignments: the likelihood of a GIVEN assignment.  Per in-span the
// feasibility code and score of its tuple (assess_in_span: the checks of V3:328-347, then the
// score_tuple() every scoring kernel uses, so a tuple of a top-K list gets its listed score bit for
// bit) and its margin against the final top-K; per service the sum of the scores and the code counts.
// The work is a gather (4E B of indices, 16E B of chosen spans per in-span), one thread per in-span.
#include "tw_kernels.cuh"

namespace tw {

__global__ void __launch_bounds__(kAssessThreads)
k_assess(tw_batch b, tw_params prm, const int32_t* __restrict__ assign, tw_score_out top, int with_top,
         AssessOut out, const int32_t* __restrict__ tile_prob, const int32_t* __restrict__ tile_start,
         double* __restrict__ tile_sum, int32_t* __restrict__ tile_cnt) {
  __shared__ double etab[64];
  __shared__ ProbView v;
  const int t = blockIdx.x, tid = threadIdx.x;
  const int p = tile_prob[t];
  if (tid == 0) load_view(b, p, v);              // the batch was validated at bind
  load_exp_table(etab);                          // its barrier also publishes v
  const int i = tile_start[t] + tid;
  int code = -1;
  double sc = 0.0;
  if (i < v.n_in) {
    const ParamView pv = param_view(prm, v, p, i / TW_PARAM_BATCH, etab);
    const int64_t gi = v.in_off + i;
    const Assessment a =
        assess_in_span(v, pv, i, assign, with_top ? top.topk_score + gi * TW_K : nullptr,
                       with_top ? top.topk_idx + TW_K * (v.tuple_off + (int64_t)i * v.E) : nullptr,
                       with_top ? top.topk_cnt[gi] : 0);
    out.score[gi] = a.score;
    out.code[gi] = (uint8_t)a.code;
    if (with_top) out.margin[gi] = a.margin;
    code = a.code;
    if (code == TW_ASSESS_SCORED) sc = a.score;
  }
  assess_tile_partials<TW_ASSESS_NCODES>(sc, code, t, tile_sum, tile_cnt);
}

// one warp per service: lane l adds tiles l, l + 32, ... in order, then a butterfly.  NC: the codes of
// the assessment kernel whose partials it adds (k_assess, k_skip_assess)
template <int NC>
__global__ void __launch_bounds__(128)
k_assess_reduce(int n_problems, const int64_t* __restrict__ prob_in_off, const int32_t* __restrict__ prob_tile0,
                const double* __restrict__ tile_sum, const int32_t* __restrict__ tile_cnt,
                double* __restrict__ prob_sum, int32_t* __restrict__ prob_count) {
  const int p = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (p >= n_problems) return;                   // warp-uniform
  const int t0 = prob_tile0[p];
  const int nt = (int)((prob_in_off[p + 1] - prob_in_off[p] + kS3Tile - 1) / kS3Tile);
  double s = 0.0;
  int cnt[NC] = {0};
  for (int k = lane; k < nt; k += 32) {
    s = dadd(s, tile_sum[t0 + k]);
#pragma unroll
    for (int q = 0; q < NC; ++q) cnt[q] += tile_cnt[(size_t)(t0 + k) * NC + q];
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    s = dadd(s, __shfl_xor_sync(kAssessAll, s, d));
#pragma unroll
    for (int q = 0; q < NC; ++q) cnt[q] += __shfl_xor_sync(kAssessAll, cnt[q], d);
  }
  if (lane == 0) {
    prob_sum[p] = s;
#pragma unroll
    for (int q = 0; q < NC; ++q) prob_count[(size_t)p * NC + q] = cnt[q];
  }
}

cudaError_t launch_assess(const tw_batch& b, const tw_params& prm, const int32_t* assign, const tw_score_out* top,
                          const AssessOut& out, const int32_t* tile_prob, const int32_t* tile_start, int n_tiles,
                          const int32_t* prob_tile0, double* tile_sum, int32_t* tile_cnt, cudaStream_t s,
                          int64_t& launches) {
  tw_score_out tk;
  memset(&tk, 0, sizeof tk);
  if (top) tk = *top;
  k_assess<<<n_tiles, kAssessThreads, 0, s>>>(b, prm, assign, tk, top != nullptr, out, tile_prob, tile_start,
                                              tile_sum, tile_cnt);
  cudaError_t e = after_launch(launches);
  if (e != cudaSuccess) return e;
  return launch_assess_reduce(TW_ASSESS_NCODES, b.n_problems, b.prob_in_off, prob_tile0, tile_sum, tile_cnt,
                              out.prob_sum, out.prob_count, s, launches);
}

cudaError_t launch_assess_reduce(int n_codes, int n_problems, const int64_t* prob_in_off, const int32_t* prob_tile0,
                                 const double* tile_sum, const int32_t* tile_cnt, double* prob_sum,
                                 int32_t* prob_count, cudaStream_t s, int64_t& launches) {
  const int warps_per_block = 128 / 32;
  const int grid = (n_problems + warps_per_block - 1) / warps_per_block;
  if (n_codes == TW_ASSESS_NCODES)
    k_assess_reduce<TW_ASSESS_NCODES><<<grid, 128, 0, s>>>(n_problems, prob_in_off, prob_tile0, tile_sum, tile_cnt,
                                                           prob_sum, prob_count);
  else
    k_assess_reduce<TW_SKIP_ASSESS_NCODES><<<grid, 128, 0, s>>>(n_problems, prob_in_off, prob_tile0, tile_sum,
                                                                tile_cnt, prob_sum, prob_count);
  return after_launch(launches);
}

}  // namespace tw
