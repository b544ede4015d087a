// tw_skip_assess.cu — tw_skip_score_assignments: the score of a GIVEN assignment of a cache-mode service.
// The skip regime's search is sequential (which skip span a tuple receives depends on every earlier
// search), but once a tuple is fixed its score depends on its own in-span only: one thread per in-span
// runs skip_assess_in_span (tw_skip_core.cuh: skip_topk's checks, then skip_score, so a listed tuple gets
// its listed score bit for bit), one CTA per 128-in-span tile; k_assess_reduce (tw_assess.cu) adds the
// tile partials per service in a fixed order.
#include "tw_kernels.cuh"
#include "tw_skip_core.cuh"

namespace tw {

// (four CTAs per SM in the bounds: ptxas then keeps the kernel free of spills across skip_score's
// division slow paths)
__global__ void __launch_bounds__(kAssessThreads, 4)
k_skip_assess(tw_batch b, tw_skip_desc sd, const int32_t* __restrict__ assign, tw_skip_out top2, int with_top,
              AssessOut out, const int32_t* __restrict__ tile_prob, const int32_t* __restrict__ tile_start,
              double* __restrict__ tile_sum, int32_t* __restrict__ tile_cnt) {
  __shared__ ProbView v;
  __shared__ SkipProb sp;
  const int t = blockIdx.x, tid = threadIdx.x;
  const int p = tile_prob[t];
  if (tid == 0) {
    load_view(b, p, v);                          // the batch was validated on the host
    sp = skip_prob(sd, v, p);
  }
  __syncthreads();
  const int i = tile_start[t] + tid;
  int code = -1;
  double sc = 0.0;
  if (i < v.n_in) {
    const int64_t gi = v.in_off + i;
    const Assessment a =
        skip_assess_in_span(v, sp, i, assign, with_top ? top2.top2_score + gi * TW_K : nullptr,
                            with_top ? top2.top2_idx + TW_K * (v.tuple_off + (int64_t)i * v.E) : nullptr,
                            with_top ? top2.top2_cnt[gi] : 0);
    out.score[gi] = a.score;
    out.code[gi] = (uint8_t)a.code;
    if (with_top) out.margin[gi] = a.margin;
    code = a.code;
    if (code == TW_ASSESS_SCORED) sc = a.score;
  }
  assess_tile_partials<TW_SKIP_ASSESS_NCODES>(sc, code, t, tile_sum, tile_cnt);
}

cudaError_t launch_skip_assess(const tw_batch& b, const tw_skip_desc& sd, const int32_t* assign, const tw_skip_out* top2,
                               const AssessOut& out, const int32_t* tile_prob, const int32_t* tile_start, int n_tiles,
                               const int32_t* prob_tile0, double* tile_sum, int32_t* tile_cnt, cudaStream_t s,
                               int64_t& launches) {
  tw_skip_out tk;
  memset(&tk, 0, sizeof tk);
  if (top2) tk = *top2;
  k_skip_assess<<<n_tiles, kAssessThreads, 0, s>>>(b, sd, assign, tk, top2 != nullptr, out, tile_prob, tile_start,
                                                   tile_sum, tile_cnt);
  cudaError_t e = after_launch(launches);
  if (e != cudaSuccess) return e;
  return launch_assess_reduce(TW_SKIP_ASSESS_NCODES, b.n_problems, b.prob_in_off, prob_tile0, tile_sum, tile_cnt,
                              out.prob_sum, out.prob_count, s, launches);
}

}  // namespace tw
