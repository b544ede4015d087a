// tw_kernels.cuh — launch-side declarations shared by the .cu files of libtw_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "tw_core.cuh"

namespace tw {

// ---- score kernel geometry (tw_score.cu) ----------------------------------------------------
constexpr int kS3Threads = 128;                  // tw_score3.cu: one CTA = one tile, one warp = 32 in-spans
constexpr int kS3Tile = 128;                     // in-spans per tile
constexpr int kStageSpans = 1536;                // out spans staged in shared memory per tile
constexpr int kTblCap = 3072;                    // term-table slots of a redo CTA (tw_score.cu)
#ifndef TW_WARP_TBL_CAP
#define TW_WARP_TBL_CAP 256
#endif
constexpr int kWarpTblCap = TW_WARP_TBL_CAP;     // term-table slots per stitch warp (search path only)
constexpr int kRedoCoopCombos = 256;             // redo kernel: in-spans with more combinations are scored by the whole warp
constexpr int kStitchCoopCombos = 512;           // in-spans with more candidate combinations are searched by the whole warp
constexpr int kTakenWords = 256;                 // taken-bitmap words a stitch warp keeps in shared memory
constexpr int kNarrowW = 2;                      // bitmap words per (in-span, ep): 64 candidates
constexpr int kWideW = 64;                       // overflow kernel: 2048 candidates per ep
constexpr int kWideThreads = 32;                 // (31 in-spans + carry-in per CTA)

// ---- stitch kernel geometry (tw_stitch.cu) --------------------------------------------------
constexpr int kStitchWarps = 2;                  // warps per CTA, one unit at a time each
// Register budget of k_stitch: 14 CTAs = 28 resident warps per SM at 72 registers.  A 64-register
// budget (32 warps) spills in the hot loop and measured slower on an H100.
constexpr int kStitchBlocksPerSM = 14;

// Term tables of the search tier (and price scratch of the warp-wide MWIS) of one stitch warp: in
// global memory, one per launched warp, so that shared memory holds only what every window touches.
struct StitchTables {
  double tbl[kWarpTblCap];
  uint8_t sid[kWarpTblCap];
};

// Per-warp shared-memory slab of k_stitch, sized per bound batch (stitch_layout): the fixed part
// (problem view, small-window solver scratch), the taken bitmap and its scratch copy sized for the
// batch's largest service (at most kTakenWords words; larger services use global memory), and the
// window buffer with the tuple planes of the batch's largest E.
struct StitchLayout {
  int tk_words;                                  // words of the taken bitmap (and of its scratch copy)
  int wb_off;                                    // byte offset of the PackedWindowBuf
  int bytes;                                     // slab bytes per warp
};
// e_max / tk_words_max: largest E and largest taken bitmap (sum over eps of n_out / 32 + 3) of the batch
StitchLayout stitch_layout(int e_max, int tk_words_max);

// Tiles: a tile never crosses a problem.  tile_prob[t], tile_start[t] (problem-local in-span).
struct TileList {
  const int32_t* tile_prob;
  const int32_t* tile_start;
  int n_tiles;
  int tile_len;
  const int32_t* tile_cnt = nullptr;   // optional explicit length per tile (<= tile_len)
};

// The scoring tiles of a bound batch, grouped by the number of eps of their problem (the scoring
// kernel is templated on E): class E occupies tiles [class_off[E-1], class_off[E]).
struct ScoreTiles {
  const int32_t* tile_prob;
  const int32_t* tile_start;
  const int32_t* tile_win;     // [n_tiles][2*TW_MAX_E]: candidate slice (first index, length) per ep
  uint8_t* overflow;           // [n_tiles] 1 = redone by the sequential kernel
  int n_tiles;
  int class_off[TW_MAX_E + 1];
};

// Kernels launched with more than 48 KB of dynamic shared memory need the limit raised once per
// device: tw_engine_create calls these for the engine's device.
cudaError_t setup_score3();                      // k_score3<1..TW_MAX_E>
cudaError_t setup_score();                       // k_score
cudaError_t setup_stitch();                      // k_stitch
cudaError_t setup_sort_ends();                   // k_sort_ends

// Every launch_* function adds the kernels it issues to `launches` (tw_engine_launch_count):
// after_launch directly follows each <<<...>>>, counts it if it was issued and returns its error.
inline cudaError_t after_launch(int64_t& launches) {
  const cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) ++launches;
  return e;
}
cudaError_t launch_prev_index(const tw_batch& b, int32_t* prev_idx, cudaStream_t s, int64_t& launches);
cudaError_t launch_tile_meta(const tw_batch& b, const TileList& tiles, int32_t* tile_win, cudaStream_t s,
                             int64_t& launches);
cudaError_t launch_score3(const tw_batch& b, const tw_params* prm, const tw_score_out& out, int keep_windows,
                          const ScoreTiles& st, const int32_t* prev_idx, cudaStream_t s, int64_t& launches);
cudaError_t launch_cut(const tw_batch& b, const tw_score_out& out, const ScoreTiles& st, const int32_t* prev_idx,
                       cudaStream_t s, int64_t& launches);
// sequential redo of the tiles the scoring kernel flagged (wide tiles subdivide scoring tiles)
cudaError_t launch_score_redo(const tw_batch& b, const tw_params* prm, const tw_score_out& out,
                              const TileList& wide, const int32_t* prev_idx, uint8_t* tile_overflow,
                              int n_sm, int* err_flag, cudaStream_t s, int64_t& launches);
// units of the stitch kernel (tw_stitch.cu: k_stitch_units): unit u = in-spans [lo[u], hi[u]) of service prob[u]
struct StitchUnits {
  int32_t* prob;
  int32_t* lo;
  int32_t* hi;
  int* count;                                    // units in the list
  int* next;                                     // queue head of k_stitch, at count + 1 (one memset resets both)
};
constexpr int kStitchUnitMin = 48;               // a unit is closed at the first strong cut after this many in-spans
constexpr int kStitchUnitsPerWarp = 6;           // large batches: longer units, about this many per resident warp
// blocks of k_stitch resident at once on the device with this slab
cudaError_t stitch_resident_blocks(const StitchLayout& layout, int n_sm, int* blocks);
// `unit_min`: shortest unit (tw_api.cu, bind); `blocks`: the persistent grid; `tables`: one
// StitchTables per warp of the grid (blocks * kStitchWarps)
cudaError_t launch_stitch(const tw_batch& b, const tw_params& prm, const uint8_t* cut,
                          const tw_score_out& spec, const tw_pass_out& out, uint32_t* taken_words, size_t taken_n_words,
                          long long node_limit, const StitchUnits& unit_buf, int unit_min, int blocks,
                          const StitchLayout& layout, StitchTables* tables, int* err_flag, cudaStream_t s,
                          int64_t& launches);
constexpr int kSortSmemCap = 16384;               // longest list the shared-memory sort network takes
cudaError_t launch_sort_ends(const tw_batch& b, int64_t* in_end_sorted, int64_t* out_end_sorted,
                             int max_seg, const int32_t* long_seg, int n_long, int64_t* long_scratch,
                             int64_t slab_len, int* err_flag, cudaStream_t s, int64_t& launches);
cudaError_t launch_params0(const tw_batch& b, const int64_t* in_end_sorted,
                           const int64_t* out_end_sorted, const int64_t* prob_gauss_off,
                           const int32_t* batch_prob, const int32_t* batch_idx, int n_batches_total,
                           double* gauss_out, const int32_t* prob_shift, cudaStream_t s, int64_t& launches);
// tw_assess.cu: one CTA per scoring tile scores the tile's given tuples and writes per-tile partial sums
// (tile_sum[t], tile_cnt[t][TW_ASSESS_NCODES]); a second kernel adds them up per service.  `top` may be
// NULL (no margin).  prob_tile0[p] = first scoring tile of problem p (its tiles are consecutive).
struct AssessOut {
  double* score;
  uint8_t* code;
  double* margin;
  double* prob_sum;
  int32_t* prob_count;
};
cudaError_t launch_assess(const tw_batch& b, const tw_params& prm, const int32_t* assign, const tw_score_out* top,
                          const AssessOut& out, const int32_t* tile_prob, const int32_t* tile_start, int n_tiles,
                          const int32_t* prob_tile0, double* tile_sum, int32_t* tile_cnt, cudaStream_t s,
                          int64_t& launches);
// tw_skip_assess.cu: the same for a cache-mode batch (tw_skip_score_assignments) over its 128-in-span tiles,
// with TW_SKIP_ASSESS_NCODES codes; `top2` may be NULL (no margin)
cudaError_t launch_skip_assess(const tw_batch& b, const tw_skip_desc& sd, const int32_t* assign, const tw_skip_out* top2,
                               const AssessOut& out, const int32_t* tile_prob, const int32_t* tile_start, int n_tiles,
                               const int32_t* prob_tile0, double* tile_sum, int32_t* tile_cnt, cudaStream_t s,
                               int64_t& launches);
// the per-service sums of either kernel's tile partials; n_codes: TW_ASSESS_NCODES or TW_SKIP_ASSESS_NCODES
cudaError_t launch_assess_reduce(int n_codes, int n_problems, const int64_t* prob_in_off, const int32_t* prob_tile0,
                                 const double* tile_sum, const int32_t* tile_cnt, double* prob_sum,
                                 int32_t* prob_count, cudaStream_t s, int64_t& launches);
constexpr int kAssessThreads = kS3Tile;          // one CTA per 128-in-span tile, one thread per in-span
constexpr unsigned kAssessAll = 0xffffffffu;
// Per-tile partials of the assessment kernels: `sc` (0 unless scored) and `code` (-1: no in-span) of every
// thread -> tile_sum[t], tile_cnt[t][NC].  A fixed order: a butterfly within each warp (every lane ends with
// the same bits), then the warps in order.
template <int NC>
__device__ __forceinline__ void assess_tile_partials(double sc, int code, int t, double* __restrict__ tile_sum,
                                                     int32_t* __restrict__ tile_cnt) {
  __shared__ double wsum[kAssessThreads / 32];
  __shared__ int wcnt[kAssessThreads / 32][NC];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) sc = dadd(sc, __shfl_xor_sync(kAssessAll, sc, d));
  int cnt[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) cnt[q] = __popc(__ballot_sync(kAssessAll, code == q));
  if (lane == 0) {
    wsum[wid] = sc;
#pragma unroll
    for (int q = 0; q < NC; ++q) wcnt[wid][q] = cnt[q];
  }
  __syncthreads();
  if (tid == 0) {
    double s = wsum[0];
    for (int w = 1; w < kAssessThreads / 32; ++w) s = dadd(s, wsum[w]);
    tile_sum[t] = s;
  }
  if (tid < NC) {
    int c = 0;
    for (int w = 0; w < kAssessThreads / 32; ++w) c += wcnt[w][tid];
    tile_cnt[(size_t)t * NC + tid] = c;
  }
}
cudaError_t launch_delays(const tw_batch& b, const int32_t* assign, const int64_t* term_sample_off,
                          const int32_t* term_ep, const int32_t* ep_prob, double* delays,
                          int32_t* counts, const int32_t* prob_shift, cudaStream_t s, int64_t& launches);

// ---- float64 timestamps (tw_times.cu): exact fixed point per problem, X = x * 2^shift[p] in int64.
// prob_shift[p] >= kShiftInvalid marks a problem with a NaN or infinite timestamp.
constexpr int kShiftInvalid = 1 << 30;
constexpr int kFixedBits = 55;                   // |X| < 2^55: differences and 100-element sums fit in int64
struct TimesF64 {
  const double* in_start;
  const double* in_end;
  const double* out_start;
  const double* out_end;
};
// prob_shift / prob_top must be zero / 0x80-byte filled; fx: [in_start | in_end | out_start | out_end] int64;
// prob_status[p] receives TW_OK, TW_ERR_INVALID (NaN / inf) or TW_ERR_RANGE_LIMIT (|X| >= 2^55).
cudaError_t launch_to_fixed(const tw_batch& b, const TimesF64& t, const int32_t* ep_prob, int32_t* prob_shift,
                            int32_t* prob_top, int64_t* fx, int32_t* prob_status, cudaStream_t s, int64_t& launches);
// scoring copy of real-unit records for a shifted batch (mode of tw_params); n_rec = records of `src`
cudaError_t launch_params_scale(int mode, const int64_t* prob_gauss_off, int n_problems, const double* src,
                                double* dst, int64_t n_rec, const int32_t* term_ep, const int32_t* ep_prob,
                                const int32_t* prob_shift, cudaStream_t s, int64_t& launches);

cudaError_t launch_gmm_prep(int n_terms, const int64_t* term_sample_off, const double* delays,
                            const int32_t* counts, int32_t* max_n, double* mean_var, cudaStream_t s,
                            int64_t& launches);
cudaError_t launch_gmm_skip(int n_problems, const int32_t* prob_ep_off, const int32_t* ep_term_off,
                            const int32_t* term_order, const int32_t* max_n,
                            const uint32_t* prob_base_skip, uint32_t* rng_skip, cudaStream_t s, int64_t& launches);
cudaError_t launch_gmm_draws(int n_problems, const int32_t* prob_ep_off, const int32_t* ep_term_off,
                             const int32_t* max_n, uint32_t* prob_draws, cudaStream_t s, int64_t& launches);
// side streams + events of the refit: the five per-K fit chains are independent and run concurrently
struct GmmFork {
  cudaStream_t side[TW_GMM_MAX_COMP] = {};
  cudaEvent_t fork = nullptr, join[TW_GMM_MAX_COMP] = {};
  bool ready = false;
  GmmFork() = default;
  GmmFork(const GmmFork&) = delete;
  GmmFork& operator=(const GmmFork&) = delete;
  ~GmmFork() {
    if (fork) cudaEventDestroy(fork);
    for (int q = 0; q < TW_GMM_MAX_COMP; ++q) {
      if (join[q]) cudaEventDestroy(join[q]);
      if (side[q]) cudaStreamDestroy(side[q]);
    }
  }
};
cudaError_t launch_gmm_fit(int n_terms, const int64_t* term_sample_off, const double* delays,
                           const int32_t* counts, const int32_t* max_n, const double* mean_var,
                           const uint32_t* rng_skip, const double* stream, int stream_len,
                           const double* stream100, double* bic, double* cen, double* mix_out,
                           int32_t* n_selected_out, int* err_flag, GmmFork* fk, cudaStream_t s,
                           int64_t& launches);

cudaError_t launch_skip(const tw_batch& b, const tw_skip_desc& sd, const tw_skip_out& out, uint32_t* taken,
                        uint32_t* set_scratch, const int64_t* prob_set_off, int32_t* win_scratch,
                        long long node_limit, int* err_flag, cudaStream_t s, int64_t& launches);
cudaError_t launch_build_dist(int n, const int64_t* ms, const int64_t* me, const int8_t* label, int E,
                              int64_t large_delay, int32_t* key, int64_t* val, cudaStream_t s, int64_t& launches);

cudaError_t launch_fp64_peak(int blocks, int iters, double* sink, cudaStream_t s, int64_t& launches);
cudaError_t gmm_work_read(unsigned long long* out, bool reset);
cudaError_t launch_in_prob(const tw_batch& b, int32_t* in_prob, cudaStream_t s, int64_t& launches);
cudaError_t launch_ground_truth(const tw_batch& b, const int32_t* in_trace, const int32_t* out_trace,
                                const int32_t* trace_lo, const int32_t* trace_n, const int64_t* tab_off, int64_t tab_len,
                                int32_t* tab, const int32_t* in_prob, int32_t* truth, cudaStream_t s,
                                int64_t& launches);
cudaError_t launch_find_order(const tw_batch& b, const int32_t* truth, const int32_t* in_prob, uint32_t* violated,
                              int* missing, cudaStream_t s, int64_t& launches);
cudaError_t launch_accuracy(const tw_batch& b, const int32_t* truth, const int32_t* assign, const int32_t* topk_idx,
                            const uint8_t* topk_cnt, const int32_t* in_trace, const int32_t* in_prob,
                            const uint8_t* prob_first, int n_traces, unsigned long long* per_prob, uint8_t* flags,
                            unsigned long long* trace_first, unsigned long long* out4, cudaStream_t s,
                            int64_t& launches);

// ---- request trees: the join (tw_traces.cu) and the analyses after it (tw_critical_path.cu,
// tw_confidence.cu).  CTAs of kTreeThreads threads; a grid-stride grid of one thread per item, at most 16
// CTAs per SM.
constexpr int kTreeThreads = 256;
inline unsigned tree_grid(int64_t n, int n_sm) {
  const int64_t want = (n + kTreeThreads - 1) / kTreeThreads;
  const int64_t cap = (int64_t)n_sm * 16;
  return (unsigned)(want < 1 ? 1 : (want < cap ? want : cap));
}

// The CTA's fixed-order sums over [lo, hi) of N double / int column pairs: v(x, s, c) adds element x into
// s[0 .. N) and c[0 .. N).  Thread t adds the elements t, t + 256, ... in order, then a butterfly per warp
// and the warps in order; thread 0 gets the sums.  ws / wc: the kernel's shared memory.
template <int N, class F>
__device__ void tree_cta_sum(int64_t lo, int64_t hi, F v, double (*ws)[kTreeThreads / 32],
                             int (*wc)[kTreeThreads / 32], double (&s)[N], int (&c)[N]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int q = 0; q < N; ++q) {
    s[q] = 0.0;
    c[q] = 0;
  }
  for (int64_t x = lo + threadIdx.x; x < hi; x += blockDim.x) v(x, s, c);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1)
    for (int q = 0; q < N; ++q) {
      s[q] = dadd(s[q], __shfl_xor_sync(0xffffffffu, s[q], d));
      c[q] += __shfl_xor_sync(0xffffffffu, c[q], d);
    }
  if (lane == 0)
    for (int q = 0; q < N; ++q) {
      ws[q][warp] = s[q];
      wc[q][warp] = c[q];
    }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < kTreeThreads / 32; ++w)
      for (int q = 0; q < N; ++q) {
        s[q] = dadd(s[q], ws[q][w]);
        c[q] += wc[q][w];
      }
  __syncthreads();
}

// tw_traces.cu: pointer-jumping rounds for n_nodes nodes, ceil(log2 n_nodes) + 1, and the launches of
// tw_assemble_traces.  claim: [n_out] scratch; err: 4 words (twice-claimed out-span, twice-named caller,
// in-span with an assign index out of range, in-span whose caller is not an out-span node: the smallest
// such node, 0x7f7f7f7f = none); changed: [rounds] flags, round r moved some node.
int trace_rounds(int64_t n_nodes);
cudaError_t launch_assemble_traces(const tw_batch& b, int64_t n_tuple, const int32_t* assign, const int32_t* in_caller,
                                   int32_t* parent, int32_t* root, int32_t* size, int32_t* claim, int32_t* err,
                                   int* changed, int rounds, int n_sm, cudaStream_t s, int64_t& launches);

// tw_critical_path.cu: the walk after the join.  Scratch per in-span: level (the level that walks it,
// -1 = none yet), window (the time type's bits), slow (its request is slow; roots only), cmax (largest
// self-time bits of the request; roots only); act: [levels] flags, level L put some in-span on the path.
// claim: the join's caller-claim words (out-span -> the in-span that names it, -1); parent: the join's
// parent words.  Any levels >= 1 gives the same results: the last level walks what lies below it.
constexpr int kCpMaxLevels = 64;
struct CpScratch {
  int32_t* level;
  int64_t* wlo;
  int64_t* whi;
  uint8_t* slow;
  unsigned long long* cmax;
  int* act;
};
cudaError_t launch_critical_paths(const tw_batch& b, const tw_times_f64* f64, const int32_t* assign,
                                  const int32_t* claim, const int32_t* parent, double slow_us,
                                  const tw_critical_out& out, const CpScratch& sc, int levels, int n_sm,
                                  cudaStream_t s, int64_t& launches);

// tw_confidence.cu: the passes after the join.  Scratch: wbits [n_in] (smallest p bits of each request),
// seg_conf / seg_req [P] (per-service partials of the batch total), flag [1] (the smallest root with
// TW_CONF_MAX_DECISIONS or more decisions, 0x7f7f7f7f = none).
struct CfScratch {
  unsigned long long* wbits;
  double* seg_conf;
  int32_t* seg_req;
  int32_t* flag;
};
cudaError_t launch_request_confidence(const tw_batch& b, const int32_t* assign, const double* score,
                                      const uint8_t* code, const tw_score_out& top, const tw_confidence_out& out,
                                      const CfScratch& sc, int n_sm, cudaStream_t s, int64_t& launches);

}  // namespace tw
