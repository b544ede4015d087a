// tw_emul_assess.cpp — k_assess (tw_assess.cu) stepped on the CPU.  TEST INFRASTRUCTURE ONLY.
//
// Compiles the engine's own assess_in_span() (tw_core.cuh) with g++ and walks the kernel's threads
// sequentially, including the order in which the kernels add the per-service sums; built by
// tests/assess_backends.py.  Not linked into libtw_b200.so.
#include <vector>

#include "../../traceweaver_b200/csrc/tw_core.cuh"

using namespace tw;

// the in-span's parameters as the kernel addresses them: the record of its 100-span batch (pass 0)
// or the problem's mixture table
static ParamView param_view(const tw_params* prm, const ProbView& v, int p, int i) {
  ParamView pv;
  pv.mode = prm->mode;
  pv.gauss = nullptr;
  pv.mix = nullptr;
  if (prm->mode == TW_PARAMS_GAUSS_BATCHED)
    pv.gauss = prm->gauss + (prm->prob_gauss_off[p] + (int64_t)(i / TW_PARAM_BATCH) * v.n_terms) * TW_GAUSS_REC;
  else
    pv.mix = prm->mix + (int64_t)v.term0 * TW_MIX_REC;
  return pv;
}

// k_assess (tw_assess.cu) for one problem: assess_in_span per in-span (thread), the tile partials and
// their per-service sum in the kernels' order (butterfly over 32 lanes, warps in order, then tile
// partials strided over 32 lanes and a butterfly).  `top` may be NULL (no margin).
static double butterfly32(double* x) {
  for (int d = 16; d > 0; d >>= 1) {
    double y[32];
    for (int l = 0; l < 32; ++l) y[l] = dadd(x[l], x[l ^ d]);
    for (int l = 0; l < 32; ++l) x[l] = y[l];
  }
  return x[0];
}

extern "C" int twe_assess_problem(const tw_batch* b, int p, const tw_params* prm, const int32_t* assign,
                                  const tw_score_out* top, double* score, uint8_t* code, double* margin,
                                  double* prob_sum, int32_t* prob_count) {
  ProbView v;
  int rc = load_view(*b, p, v);
  if (rc) return rc;
  const int n_tiles = (v.n_in + 127) / 128;
  std::vector<double> tile_sum((size_t)n_tiles);
  for (int q = 0; q < TW_ASSESS_NCODES; ++q) prob_count[(size_t)p * TW_ASSESS_NCODES + q] = 0;
  for (int t = 0; t < n_tiles; ++t) {
    double wsum[4];
    for (int w = 0; w < 4; ++w) {
      double lanes[32];
      for (int l = 0; l < 32; ++l) {
        const int i = t * 128 + w * 32 + l;
        lanes[l] = 0.0;
        if (i >= v.n_in) continue;
        const ParamView pv = param_view(prm, v, p, i);
        const int64_t gi = v.in_off + i;
        const Assessment a = assess_in_span(v, pv, i, assign, top ? top->topk_score + gi * TW_K : nullptr,
                                            top ? top->topk_idx + TW_K * (v.tuple_off + (int64_t)i * v.E) : nullptr,
                                            top ? top->topk_cnt[gi] : 0);
        score[gi] = a.score;
        code[gi] = (uint8_t)a.code;
        if (top) margin[gi] = a.margin;
        prob_count[(size_t)p * TW_ASSESS_NCODES + a.code] += 1;
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
