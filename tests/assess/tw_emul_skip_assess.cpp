// tw_emul_skip_assess.cpp — k_skip_assess (tw_skip_assess.cu) stepped on the CPU.  TEST INFRASTRUCTURE ONLY.
//
// Compiles the engine's own skip_assess_in_span() (tw_skip_core.cuh) with g++ and walks the kernel's
// threads sequentially, with the per-service sums in the kernels' order (tw_emul_assess.cpp, included
// for its butterfly); built by tests/assess/skip_emul_assess.py.  Not linked into libtw_b200.so.
#include "tw_emul_assess.cpp"
#include "../../traceweaver_b200/csrc/tw_skip_core.cuh"

// k_skip_assess for one problem; `top2` may be NULL (no margin)
extern "C" int twe_skip_assess_problem(const tw_batch* b, int p, const tw_skip_desc* sd, const int32_t* assign,
                                       const tw_skip_out* top2, double* score, uint8_t* code, double* margin,
                                       double* prob_sum, int32_t* prob_count) {
  ProbView v;
  int rc = load_view(*b, p, v);
  if (rc) return rc;
  const SkipProb sp = skip_prob(*sd, v, p);
  const int n_tiles = (v.n_in + 127) / 128;
  std::vector<double> tile_sum((size_t)n_tiles);
  for (int q = 0; q < TW_SKIP_ASSESS_NCODES; ++q) prob_count[(size_t)p * TW_SKIP_ASSESS_NCODES + q] = 0;
  for (int t = 0; t < n_tiles; ++t) {
    double wsum[4];
    for (int w = 0; w < 4; ++w) {
      double lanes[32];
      for (int l = 0; l < 32; ++l) {
        const int i = t * 128 + w * 32 + l;
        lanes[l] = 0.0;
        if (i >= v.n_in) continue;
        const int64_t gi = v.in_off + i;
        const Assessment a =
            skip_assess_in_span(v, sp, i, assign, top2 ? top2->top2_score + gi * TW_K : nullptr,
                                top2 ? top2->top2_idx + TW_K * (v.tuple_off + (int64_t)i * v.E) : nullptr,
                                top2 ? top2->top2_cnt[gi] : 0);
        score[gi] = a.score;
        code[gi] = (uint8_t)a.code;
        if (top2) margin[gi] = a.margin;
        prob_count[(size_t)p * TW_SKIP_ASSESS_NCODES + a.code] += 1;
        if (a.code == TW_ASSESS_SCORED) lanes[l] = a.score;
      }
      wsum[w] = butterfly32(lanes);
    }
    double s = wsum[0];
    for (int w = 1; w < 4; ++w) s = dadd(s, wsum[w]);
    tile_sum[t] = s;
  }
  double lanes[32];
  for (int l = 0; l < 32; ++l) {
    lanes[l] = 0.0;
    for (int k = l; k < n_tiles; k += 32) lanes[l] = dadd(lanes[l], tile_sum[k]);
  }
  prob_sum[p] = butterfly32(lanes);
  return TW_OK;
}
