// tw_api.cu — the C ABI of libtw_b200.so (include/traceweaver_b200.h): engine object, batch
// binding (validation, tile lists, scratch), and the entry points that launch the kernels.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "tw_kernels.cuh"

using namespace tw;

static thread_local std::string g_last_error;

static int fail(int code, const char* fmt, const char* a = "", const char* b2 = "") {
  char buf[512];
  snprintf(buf, sizeof buf, fmt, a, b2);
  g_last_error = buf;
  return code;
}

#define CU(expr)                                                                      \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) return fail(TW_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

// Device scratch owned by the engine, grow-only: re-binding a batch of similar size allocates nothing.
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  // room for `count` elements (1 if 0), with 1/8 headroom when it has to grow.  A reallocation loses
  // the contents: `valid`, the flag of a cache kept in this buffer, is cleared then.
  cudaError_t reserve(size_t count, bool* valid = nullptr) {
    const size_t need = (count ? count : 1) * sizeof(T);
    if (bytes >= need) return cudaSuccess;
    if (valid) *valid = false;
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
    const size_t cap = need + need / 8;
    cudaError_t e = cudaMalloc((void**)&p, cap);
    if (e != cudaSuccess) return e;
    bytes = cap;
    return cudaSuccess;
  }
};

struct tw_engine {
  int device = 0;
  int n_sm = 0;
  bool bound = false;
  tw_batch dev{};
  int64_t launches = 0;
  // host descriptors
  std::vector<int64_t> prob_in_off;
  std::vector<int32_t> prob_ep_off;
  int max_seg = 0;
  int64_t dev_n_tuple = 0;
  // device status word: allocated and zeroed with the engine, sticky across re-binds (a caller that
  // pipelines several batches through one engine reads it once at the end), cleared by tw_engine_status only
  DevBuf<int> err_flag;
  DevBuf<int32_t> prev_idx;
  DevBuf<int32_t> score_tiles;       // [2*n]: prob, start; grouped by the problem's E (class_off)
  DevBuf<int32_t> tile_win;          // [n][2*TW_MAX_E] candidate slice per ep (k_tile_meta)
  DevBuf<int32_t> wide_tiles;        // [4*n]: prob, start, scoring-tile index, length
  int n_tiles = 0, n_wide = 0;
  int class_off[TW_MAX_E + 1] = {0};
  // tw_score_assignments: first scoring tile of every problem (host list built at bind, uploaded on
  // first use) and the per-tile partial sums
  std::vector<int32_t> prob_tile0;
  bool prob_tile0_uploaded = false;
  DevBuf<int32_t> assess_tile0;
  DevBuf<double> assess_tile_sum;
  DevBuf<int32_t> assess_tile_cnt;
  DevBuf<uint8_t> tile_overflow;
  bool windows_valid = false;        // cut / maps / overflow flags of this batch have been produced
  DevBuf<int32_t> own_used_lo;       // candidate maps when the caller does not ask for them
  DevBuf<uint32_t> own_used_bits;
  DevBuf<uint8_t> own_used_wide;
  DevBuf<uint32_t> taken;
  size_t taken_words = 0;
  DevBuf<double> fp64_sink;          // tw_measure_fp64_peak
  // ground truth / order / accuracy scratch (tw_truth.cu)
  DevBuf<int32_t> truth_tab;
  DevBuf<int64_t> truth_tab_off;
  DevBuf<int32_t> in_prob;
  DevBuf<int> order_missing;
  DevBuf<uint8_t> acc_flags;
  DevBuf<unsigned long long> acc_first;
  // request trees (tw_assemble_traces): caller claim words, error words + per-round flags, the parent and
  // size words of a join whose caller keeps only the roots (tw_critical_paths, tw_request_confidence), and
  // what the last call did (tw_debug_trace_rounds)
  DevBuf<int32_t> trace_claim;
  DevBuf<int32_t> trace_flags;
  DevBuf<int32_t> trace_parent;
  DevBuf<int32_t> trace_size;
  int trace_rounds_launched = 0, trace_rounds_run = 0, trace_still = 0;
  // critical paths (tw_critical_paths): the walk's scratch (CpScratch), the level launches of the last call
  // (tw_debug_critical_levels) and a forced level count, 0 = from the rounds (tw_debug_critical_force_levels)
  DevBuf<int32_t> cp_level;
  DevBuf<int64_t> cp_wlo;
  DevBuf<int64_t> cp_whi;
  DevBuf<uint8_t> cp_slow;
  DevBuf<unsigned long long> cp_cmax;
  DevBuf<int> cp_act;
  int cp_levels = 0, cp_force_levels = 0;
  // request confidence (tw_request_confidence): CfScratch
  DevBuf<unsigned long long> cf_wbits;
  DevBuf<double> cf_seg_conf;
  DevBuf<int32_t> cf_seg_req;
  DevBuf<int32_t> cf_flag;
  // skip / cache mode scratch (tw_skip_solve)
  DevBuf<uint32_t> skip_sets;
  DevBuf<int64_t> skip_set_off;
  DevBuf<uint32_t> skip_taken;
  DevBuf<int32_t> skip_win;
  DevBuf<int32_t> skip_tiles;        // tw_skip_score_assignments: tile prob, tile start, first tile per problem
  DevBuf<double> skip_tile_sum;      // and the per-tile partials
  DevBuf<int32_t> skip_tile_cnt;
  DevBuf<int32_t> unit_prob;         // stitch units (k_stitch_units)
  DevBuf<int32_t> unit_lo;
  DevBuf<int32_t> unit_hi;
  DevBuf<int> unit_count;
  int max_units = 0;
  int unit_min = kStitchUnitMin;     // shortest unit of the bound batch (bind)
  StitchLayout stitch_layout{};      // per-warp shared memory of k_stitch for the bound batch
  int stitch_blocks = 0;             // persistent grid of k_stitch (bind; tw_debug_stitch_grid)
  int stitch_blocks_max = 0;         // the grid the bind sized stitch_tables for
  DevBuf<StitchTables> stitch_tables;   // search tables, one per warp of the grid
  DevBuf<int32_t> long_seg;          // lists longer than kSortSmemCap (sorted in global memory)
  int n_long = 0;
  DevBuf<int64_t> long_scratch;
  int64_t slab_len = 1;
  DevBuf<int64_t> in_end_sorted;
  DevBuf<int64_t> out_end_sorted;
  DevBuf<int32_t> batch_prob;
  DevBuf<int32_t> batch_idx;
  int n_batches_total = 0;
  DevBuf<int32_t> term_ep;
  DevBuf<int32_t> ep_prob;
  // float64 timestamps (tw_engine_bind_f64): the fixed-point copies the kernels read, the shift of every
  // problem, and the scoring copy of the parameter records (k_params_scale)
  bool shifted = false;
  DevBuf<int64_t> fixed_times;
  DevBuf<int32_t> prob_shift;
  DevBuf<int32_t> prob_top;
  DevBuf<int32_t> prob_status;
  DevBuf<double> scaled_params;
  int64_t n_gauss_rec = 0;
  long long node_limit = 2000000LL;   // exact MWIS search nodes per window before TW_ERR_MWIS_LIMIT
  // refit scratch (allocated on first tw_gmm_refit after bind)
  static constexpr int kStreamLen = 16384;
  DevBuf<int32_t> gmm_max_n;
  DevBuf<double> gmm_mean_var;
  DevBuf<uint32_t> gmm_skip;
  DevBuf<double> gmm_bic;
  DevBuf<double> gmm_cen;         // k-means centres handed from the seeding to the Lloyd to the EM kernels
  GmmFork gmm_fork;               // side streams of the five per-K fit chains
  DevBuf<double> gmm_stream;
  DevBuf<double> gmm_stream100;
  uint32_t gmm_seed = 0;
  bool gmm_seed_valid = false;    // gmm_stream holds the draws of gmm_seed
  bool gmm_stream100_valid = false;
};

extern "C" {

int tw_abi_version(void) { return TW_ABI_VERSION; }

const char* tw_last_error(void) { return g_last_error.c_str(); }

int tw_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int tw_engine_create(int device, tw_engine** out) {
  if (!out) return fail(TW_ERR_INVALID, "tw_engine_create: out is NULL");
  int n = tw_device_count();
  if (device < 0 || device >= n) return fail(TW_ERR_NO_DEVICE, "tw_engine_create: no CUDA device %s", "");
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, device));
  // arch-specific sm_90a code loads on compute capability 9.0 only
  if (prop.major != 9 || prop.minor != 0)
    return fail(TW_ERR_NO_DEVICE, "tw_engine_create: built for sm_90a (H100), found %s", prop.name);
  CU(cudaSetDevice(device));
  CU(setup_score3());
  CU(setup_score());
  CU(setup_stitch());
  CU(setup_sort_ends());
  std::unique_ptr<tw_engine> e(new tw_engine);
  e->device = device;
  e->n_sm = prop.multiProcessorCount;
  CU(e->err_flag.reserve(1));
  CU(cudaMemset(e->err_flag.p, 0, sizeof(int)));
  CU(cudaDeviceSynchronize());   // cudaMemset is asynchronous, and the kernels run on the caller's streams
  *out = e.release();
  return TW_OK;
}

int tw_engine_destroy(tw_engine* eng) {
  if (!eng) return TW_OK;
  cudaSetDevice(eng->device);
  delete eng;
  return TW_OK;
}

// Host-side checks of a batch descriptor.  Every entry point checks the offset tables and the totals.
// With `terms` (the entry points that solve) also the term lists and the DAG, >= 2 incoming spans per
// problem and non-empty outgoing lists; outgoing lists must then be as long as the incoming list
// unless `allow_skip` (tw_skip_solve).
static int validate_host(const tw_batch* h, const char* who, bool terms, bool allow_skip) {
  if (!h || h->n_problems < 1) return fail(TW_ERR_INVALID, "%s: no problems", who);
  if (!h->prob_in_off || !h->prob_ep_off || !h->prob_tuple_off || !h->ep_out_off ||
      (terms && (!h->ep_term_off || !h->ep_pred_mask || !h->term_src)))
    return fail(TW_ERR_INVALID, "%s: NULL descriptor array", who);
  const int P = h->n_problems;
  if (h->prob_in_off[0] != 0 || h->prob_ep_off[0] != 0 || h->prob_tuple_off[0] != 0 || h->ep_out_off[0] != 0 ||
      (terms && h->ep_term_off[0] != 0))
    return fail(TW_ERR_INVALID, "%s: offsets must start at 0", who);
  for (int p = 0; p < P; ++p) {
    int E = h->prob_ep_off[p + 1] - h->prob_ep_off[p];
    int64_t n = h->prob_in_off[p + 1] - h->prob_in_off[p];
    if (E < 1 || E > TW_MAX_E) return fail(TW_ERR_INVALID, "%s: E outside [1, TW_MAX_E]", who);
    if (n < (terms ? 2 : 1) || n > 0x7fffffff) return fail(TW_ERR_INVALID, "%s: incoming span count out of range", who);
    if (h->prob_tuple_off[p + 1] - h->prob_tuple_off[p] != n * E)
      return fail(TW_ERR_INVALID, "%s: prob_tuple_off inconsistent", who);
    if (!terms) continue;
    int ep0 = h->prob_ep_off[p];
    int nt = h->ep_term_off[ep0 + E] - h->ep_term_off[ep0];
    if (nt < E || nt > TW_MAX_TERMS) return fail(TW_ERR_INVALID, "%s: term count out of range", who);
    for (int e = 0; e < E; ++e) {
      int64_t no = h->ep_out_off[ep0 + e + 1] - h->ep_out_off[ep0 + e];
      if (no != n && !allow_skip)
        return fail(TW_ERR_UNSUPPORTED, "%s: n_out != n_in (skip budgets): use tw_skip_solve for this service", who);
      if (no < 1) return fail(TW_ERR_INVALID, "%s: an outgoing list is empty", who);
      uint32_t pm = h->ep_pred_mask[ep0 + e];
      if (pm >> e) return fail(TW_ERR_INVALID, "%s: predecessor mask must reference earlier eps only", who);
      int t0 = h->ep_term_off[ep0 + e], t1 = h->ep_term_off[ep0 + e + 1];
      if (t1 <= t0 || h->term_src[t1 - 1] != TW_TERM_LAST) return fail(TW_ERR_INVALID, "%s: ep terms must end with LAST", who);
      for (int t = t0; t < t1 - 1; ++t) {
        int src = h->term_src[t];
        if (src == TW_TERM_ROOT) { if (pm) return fail(TW_ERR_INVALID, "%s: ROOT term on an ep with in-edges", who); }
        else if (src < 0 || src >= e || !(pm >> src & 1u)) return fail(TW_ERR_INVALID, "%s: edge term without DAG edge", who);
      }
    }
  }
  if (h->prob_in_off[P] != h->n_in_total || h->prob_ep_off[P] != h->n_ep_total ||
      h->ep_out_off[h->n_ep_total] != h->n_out_total || (terms && h->ep_term_off[h->n_ep_total] != h->n_term_total))
    return fail(TW_ERR_INVALID, "%s: totals inconsistent", who);
  return TW_OK;
}

int tw_batch_validate_host(const tw_batch* h) { return validate_host(h, "batch", true, false); }

int tw_engine_bind(tw_engine* eng, const tw_batch* dev, const tw_batch* h, void* stream_) {
  if (!eng || !dev || !h) return fail(TW_ERR_INVALID, "tw_engine_bind: NULL argument");
  cudaStream_t s = (cudaStream_t)stream_;
  int rc = tw_batch_validate_host(h);
  if (rc) return rc;
  CU(cudaSetDevice(eng->device));
  eng->bound = false;
  eng->shifted = false;
  eng->dev = *dev;
  const int P = h->n_problems;
  eng->prob_in_off.assign(h->prob_in_off, h->prob_in_off + P + 1);
  eng->prob_ep_off.assign(h->prob_ep_off, h->prob_ep_off + P + 1);
  eng->dev_n_tuple = h->prob_tuple_off[P];

  // ---- tile lists (a tile never crosses a problem; scoring tiles are grouped by E; wide tiles
  // subdivide scoring tiles and carry their length)
  std::vector<int32_t> nt_prob, nt_start, wt_prob, wt_start, wt_narrow, wt_len, bprob, bidx;
  const int wide_len = kWideThreads - 1;
  int64_t n_gauss_rec = 0;
  eng->max_seg = 0;
  eng->windows_valid = false;
  eng->class_off[0] = 0;
  eng->prob_tile0.assign((size_t)P, 0);
  eng->prob_tile0_uploaded = false;
  for (int Ec = 1; Ec <= TW_MAX_E; ++Ec) {
    for (int p = 0; p < P; ++p) {
      if (h->prob_ep_off[p + 1] - h->prob_ep_off[p] != Ec) continue;
      int n = (int)(h->prob_in_off[p + 1] - h->prob_in_off[p]);
      for (int i0 = 0; i0 < n; i0 += kS3Tile) {
        int tile_id = (int)nt_prob.size();
        if (i0 == 0) eng->prob_tile0[p] = tile_id;
        nt_prob.push_back(p);
        nt_start.push_back(i0);
        int lim = i0 + kS3Tile < n ? i0 + kS3Tile : n;
        for (int j0 = i0; j0 < lim; j0 += wide_len) {
          wt_prob.push_back(p);
          wt_start.push_back(j0);
          wt_narrow.push_back(tile_id);
          wt_len.push_back(lim - j0 < wide_len ? lim - j0 : wide_len);
        }
      }
    }
    eng->class_off[Ec] = (int)nt_prob.size();
  }
  for (int p = 0; p < P; ++p) {
    int n = (int)(h->prob_in_off[p + 1] - h->prob_in_off[p]);
    if (n > eng->max_seg) eng->max_seg = n;
    int nb = (n + TW_PARAM_BATCH - 1) / TW_PARAM_BATCH;
    for (int q = 0; q < nb; ++q) { bprob.push_back(p); bidx.push_back(q); }
    const int ep0 = h->prob_ep_off[p];
    n_gauss_rec += (int64_t)nb * (h->ep_term_off[h->prob_ep_off[p + 1]] - h->ep_term_off[ep0]);
  }
  eng->n_tiles = (int)nt_prob.size();
  eng->n_wide = (int)wt_prob.size();
  eng->n_batches_total = (int)bprob.size();
  eng->n_gauss_rec = n_gauss_rec;
  std::vector<int32_t> term_ep(h->n_term_total), ep_prob(h->n_ep_total);
  for (int p = 0; p < P; ++p)
    for (int ep = h->prob_ep_off[p]; ep < h->prob_ep_off[p + 1]; ++ep) {
      ep_prob[ep] = p;
      for (int t = h->ep_term_off[ep]; t < h->ep_term_off[ep + 1]; ++t) term_ep[t] = ep;
    }

  CU(eng->prev_idx.reserve((size_t)h->n_in_total));
  CU(eng->score_tiles.reserve((size_t)eng->n_tiles * 2));
  CU(eng->tile_win.reserve((size_t)eng->n_tiles * 2 * TW_MAX_E));
  CU(eng->wide_tiles.reserve((size_t)eng->n_wide * 4));
  CU(eng->tile_overflow.reserve((size_t)eng->n_tiles));
  eng->taken_words = (size_t)(h->n_out_total / 32) + (size_t)h->n_ep_total + 2;
  CU(eng->taken.reserve(eng->taken_words));
  CU(eng->in_end_sorted.reserve((size_t)h->n_in_total));
  CU(eng->out_end_sorted.reserve((size_t)h->n_out_total));
  CU(eng->batch_prob.reserve(bprob.size()));
  CU(eng->batch_idx.reserve(bidx.size()));
  CU(eng->term_ep.reserve(term_ep.size()));
  CU(eng->ep_prob.reserve(ep_prob.size()));
  auto up = [&](void* dst, const std::vector<int32_t>& src) {
    return cudaMemcpyAsync(dst, src.data(), src.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s);
  };
  CU(up(eng->score_tiles.p, nt_prob));
  CU(up(eng->score_tiles.p + eng->n_tiles, nt_start));
  CU(up(eng->wide_tiles.p, wt_prob));
  CU(up(eng->wide_tiles.p + eng->n_wide, wt_start));
  CU(up(eng->wide_tiles.p + 2 * eng->n_wide, wt_narrow));
  CU(up(eng->wide_tiles.p + 3 * eng->n_wide, wt_len));
  CU(up(eng->batch_prob.p, bprob));
  CU(up(eng->batch_idx.p, bidx));
  CU(up(eng->term_ep.p, term_ep));
  CU(up(eng->ep_prob.p, ep_prob));
  CU(cudaStreamSynchronize(s));   // staging vectors go out of scope

  // shared-memory slab of a stitch warp: sized for the batch's largest E and largest taken bitmap
  int stitch_resident = 0;   // blocks of k_stitch the device holds at once with this slab
  {
    int e_max = 1, tk_max = 0;
    for (int p = 0; p < P; ++p) {
      const int ep0 = h->prob_ep_off[p], E = h->prob_ep_off[p + 1] - ep0;
      int tk = 0;
      for (int e = 0; e < E; ++e) tk += (int)((h->ep_out_off[ep0 + e + 1] - h->ep_out_off[ep0 + e]) >> 5) + 3;
      e_max = E > e_max ? E : e_max;
      tk_max = tk > tk_max ? tk : tk_max;
    }
    eng->stitch_layout = stitch_layout(e_max, tk_max);
    CU(stitch_resident_blocks(eng->stitch_layout, eng->n_sm, &stitch_resident));
  }
  // unit list of the stitch kernel: at most n / unit_min + 1 units per service.  Every unit pays a
  // set-up (problem view, bitmap, defaults, cold records), so a large batch takes longer units: about
  // kStitchUnitsPerWarp per resident warp, which still leaves the queue enough units to end the pass
  // on a short tail.
  {
    const int64_t per_batch = h->n_in_total / ((int64_t)kStitchUnitsPerWarp * stitch_resident * kStitchWarps);
    eng->unit_min = per_batch > kStitchUnitMin ? (int)per_batch : kStitchUnitMin;
    int64_t mu = 0;
    for (int p = 0; p < P; ++p) mu += (h->prob_in_off[p + 1] - h->prob_in_off[p]) / eng->unit_min + 1;
    if (mu > 0x7fffffff) return fail(TW_ERR_RANGE_LIMIT, "bind: too many stitch units");
    eng->max_units = (int)mu;
    CU(eng->unit_prob.reserve((size_t)mu));
    CU(eng->unit_lo.reserve((size_t)mu));
    CU(eng->unit_hi.reserve((size_t)mu));
    CU(eng->unit_count.reserve(2));
    // the persistent grid: every resident block, or one warp per unit if the list is shorter
    const int64_t needed = (mu + kStitchWarps - 1) / kStitchWarps;
    eng->stitch_blocks = (int)(needed < stitch_resident ? needed : stitch_resident);
    eng->stitch_blocks_max = eng->stitch_blocks;
    CU(eng->stitch_tables.reserve((size_t)eng->stitch_blocks * kStitchWarps));
  }
  // lists too long for the shared-memory sort of tw_prepare get a slab of global scratch each
  {
    std::vector<int32_t> long_seg;
    int64_t longest = 0;
    for (int p = 0; p < P; ++p) {
      const int64_t n = h->prob_in_off[p + 1] - h->prob_in_off[p];
      if (n > kSortSmemCap) { long_seg.push_back(p); longest = n > longest ? n : longest; }
    }
    for (int ep = 0; ep < h->n_ep_total; ++ep) {
      const int64_t n = h->ep_out_off[ep + 1] - h->ep_out_off[ep];
      if (n > kSortSmemCap) { long_seg.push_back(P + ep); longest = n > longest ? n : longest; }
      if (n > eng->max_seg) eng->max_seg = (int)n;
    }
    if (longest > (int64_t)1 << 28) return fail(TW_ERR_RANGE_LIMIT, "bind: a list has more than 2^28 spans");
    eng->n_long = (int)long_seg.size();
    eng->slab_len = 1;
    while (eng->slab_len < longest) eng->slab_len <<= 1;
    CU(eng->long_seg.reserve(long_seg.size()));
    CU(eng->long_scratch.reserve((size_t)eng->n_long * (size_t)eng->slab_len));
    if (eng->n_long) {
      CU(cudaMemcpyAsync(eng->long_seg.p, long_seg.data(), long_seg.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
      CU(cudaStreamSynchronize(s));
    }
  }
  eng->bound = true;
  return TW_OK;
}

int tw_engine_bind_f64(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const tw_times_f64* times,
                       void* stream_) {
  if (!eng || !dev || !h || !times || !times->in_start || !times->in_end || !times->out_start || !times->out_end)
    return fail(TW_ERR_INVALID, "tw_engine_bind_f64: NULL argument");
  int rc = tw_engine_bind(eng, dev, h, stream_);
  if (rc) return rc;
  eng->bound = false;
  cudaStream_t s = (cudaStream_t)stream_;
  const int P = h->n_problems;
  const size_t n_in = (size_t)h->n_in_total, n_out = (size_t)h->n_out_total;
  CU(eng->fixed_times.reserve(2 * (n_in + n_out)));
  CU(eng->prob_shift.reserve((size_t)P));
  CU(eng->prob_top.reserve((size_t)P));
  CU(eng->prob_status.reserve((size_t)P));
  CU(cudaMemsetAsync(eng->prob_shift.p, 0, (size_t)P * sizeof(int32_t), s));
  CU(cudaMemsetAsync(eng->prob_top.p, 0x80, (size_t)P * sizeof(int32_t), s));   // below every floor(log2 |x|)
  TimesF64 t{times->in_start, times->in_end, times->out_start, times->out_end};
  CU(launch_to_fixed(eng->dev, t, eng->ep_prob.p, eng->prob_shift.p, eng->prob_top.p, eng->fixed_times.p,
                     eng->prob_status.p, s, eng->launches));
  std::vector<int32_t> status((size_t)P);
  CU(cudaMemcpyAsync(status.data(), eng->prob_status.p, (size_t)P * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  for (int p = 0; p < P; ++p) {
    if (status[p] == TW_OK) continue;
    char which[32];
    snprintf(which, sizeof which, "%d", p);
    return fail(status[p], status[p] == TW_ERR_INVALID
                               ? "tw_engine_bind_f64: problem %s has a NaN or infinite timestamp"
                               : "tw_engine_bind_f64: problem %s needs more than 55 bits in fixed point%s",
                which, status[p] == TW_ERR_INVALID ? "" : " (magnitude x resolution of its timestamps too large)");
  }
  int64_t* fx = eng->fixed_times.p;
  eng->dev.in_start = fx;
  eng->dev.in_end = fx + n_in;
  eng->dev.out_start = fx + 2 * n_in;
  eng->dev.out_end = fx + 2 * n_in + n_out;
  eng->shifted = true;
  eng->bound = true;
  return TW_OK;
}

// For a shifted batch the scoring kernels read a rescaled copy of the caller's real-unit records.
static int scoring_params(tw_engine* eng, const tw_params* params, tw_params& scaled, cudaStream_t s) {
  scaled = *params;
  if (!eng->shifted) return TW_OK;
  const bool gauss = params->mode == TW_PARAMS_GAUSS_BATCHED;
  const int64_t n_rec = gauss ? eng->n_gauss_rec : eng->dev.n_term_total;
  const size_t width = gauss ? TW_GAUSS_REC : TW_MIX_REC;
  CU(eng->scaled_params.reserve((size_t)n_rec * width));
  CU(launch_params_scale(params->mode, params->prob_gauss_off, eng->dev.n_problems, gauss ? params->gauss : params->mix,
                         eng->scaled_params.p, n_rec, eng->term_ep.p, eng->ep_prob.p, eng->prob_shift.p, s,
                         eng->launches));
  if (gauss) scaled.gauss = eng->scaled_params.p;
  else scaled.mix = eng->scaled_params.p;
  return TW_OK;
}

int tw_prepare(tw_engine* eng, void* stream_) {
  if (!eng || !eng->bound) return fail(TW_ERR_INVALID, "tw_prepare: no batch bound");
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  CU(launch_prev_index(eng->dev, eng->prev_idx.p, s, eng->launches));
  CU(launch_sort_ends(eng->dev, eng->in_end_sorted.p, eng->out_end_sorted.p, eng->max_seg, eng->long_seg.p, eng->n_long,
                      eng->long_scratch.p, eng->slab_len, eng->err_flag.p, s, eng->launches));
  TileList tl{eng->score_tiles.p, eng->score_tiles.p + eng->n_tiles, eng->n_tiles, kS3Tile};
  CU(launch_tile_meta(eng->dev, tl, eng->tile_win.p, s, eng->launches));
  return TW_OK;
}

int tw_engine_status(tw_engine* eng, void* stream_) {
  if (!eng) return fail(TW_ERR_INVALID, "tw_engine_status: NULL engine");
  cudaStream_t s = (cudaStream_t)stream_;
  int flag = 0;
  CU(cudaMemcpyAsync(&flag, eng->err_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (flag != 0) {
    CU(cudaMemsetAsync(eng->err_flag.p, 0, sizeof(int), s));
    return fail(flag, "device-side status %s", flag == TW_ERR_MWIS_LIMIT ? "TW_ERR_MWIS_LIMIT"
                                               : flag == TW_ERR_RANGE_LIMIT ? "TW_ERR_RANGE_LIMIT"
                                               : flag == TW_ERR_REFERENCE_UNDEFINED ? "TW_ERR_REFERENCE_UNDEFINED" : "error");
  }
  return TW_OK;
}

int64_t tw_engine_launch_count(const tw_engine* eng) { return eng ? eng->launches : 0; }

int tw_engine_tile_stats(tw_engine* eng, int64_t* n_tiles, int64_t* n_redone, void* stream_) {
  if (!eng || !eng->bound) return fail(TW_ERR_INVALID, "tw_engine_tile_stats: no batch bound");
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  if (n_tiles) *n_tiles = eng->n_tiles;
  if (n_redone) {
    std::vector<uint8_t> h((size_t)eng->n_tiles);
    *n_redone = 0;
    if (eng->windows_valid) {
      CU(cudaMemcpyAsync(h.data(), eng->tile_overflow.p, h.size(), cudaMemcpyDeviceToHost, s));
      CU(cudaStreamSynchronize(s));
      for (uint8_t f : h) *n_redone += f != 0;
    }
  }
  return TW_OK;
}

int tw_skip_solve(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const tw_skip_desc* sd, const tw_skip_out* out,
                  void* stream_) {
  if (!eng || !dev || !h || !sd || !out) return fail(TW_ERR_INVALID, "tw_skip_solve: NULL argument");
  int rc = validate_host(h, "batch", true, true);
  if (rc) return rc;
  if (!out->pass.assign || !out->pass.mis_rank || !out->pass.n_cand || !out->pass.counters || !out->top2_score ||
      !out->top2_idx || !out->top2_cnt || !out->cut)
    return fail(TW_ERR_INVALID, "tw_skip_solve: NULL output array");
  if ((out->pass.topk_score != nullptr) != (out->pass.topk_idx != nullptr) ||
      (out->pass.topk_score != nullptr) != (out->pass.topk_cnt != nullptr))
    return fail(TW_ERR_INVALID, "tw_skip_solve: topk_* must be all set or all NULL");
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  const int P = h->n_problems;
  // candidate-set bitmaps: three per problem, one word-aligned stretch per ep
  std::vector<int64_t> set_off((size_t)P + 1, 0);
  for (int p = 0; p < P; ++p) {
    int64_t words = 0;
    for (int ep = h->prob_ep_off[p]; ep < h->prob_ep_off[p + 1]; ++ep)
      words += (h->ep_out_off[ep + 1] - h->ep_out_off[ep] + 31) / 32;
    set_off[p + 1] = set_off[p] + words;
  }
  CU(eng->skip_sets.reserve((size_t)(3 * set_off[P])));
  CU(eng->skip_set_off.reserve((size_t)P + 1));
  CU(eng->skip_taken.reserve((size_t)(h->n_out_total / 32) + (size_t)h->n_ep_total + 2));
  // per (ep, window) prefix + fetch counters: the host does not know prob_cnt_off (device array), so
  // size it by an upper bound the caller's skip_count array must respect: read the last offset
  int64_t cnt_total = 0;
  CU(cudaMemcpyAsync(&cnt_total, sd->prob_cnt_off + P, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (cnt_total < 0) return fail(TW_ERR_INVALID, "tw_skip_solve: prob_cnt_off inconsistent");
  CU(eng->skip_win.reserve((size_t)(2 * cnt_total)));
  CU(cudaMemcpyAsync(eng->skip_set_off.p, set_off.data(), set_off.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  CU(launch_skip(*dev, *sd, *out, eng->skip_taken.p, eng->skip_sets.p, eng->skip_set_off.p, eng->skip_win.p,
                 eng->node_limit, eng->err_flag.p, s, eng->launches));
  CU(cudaStreamSynchronize(s));    // set_off goes out of scope
  return TW_OK;
}

int tw_skip_score_assignments(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const tw_skip_desc* sd,
                              const int32_t* assign, const tw_skip_out* top2, double* score_out, uint8_t* code_out,
                              double* margin_out, double* prob_sum_out, int32_t* prob_count_out, void* stream_) {
  if (!eng || !dev || !h || !sd || !assign || !score_out || !code_out || !prob_sum_out || !prob_count_out)
    return fail(TW_ERR_INVALID, "tw_skip_score_assignments: NULL argument");
  if ((top2 != nullptr) != (margin_out != nullptr))
    return fail(TW_ERR_INVALID, "tw_skip_score_assignments: top2 and margin_out go together");
  if (top2 && (!top2->top2_score || !top2->top2_idx || !top2->top2_cnt))
    return fail(TW_ERR_INVALID, "tw_skip_score_assignments: top2 needs top2_score, top2_idx and top2_cnt");
  int rc = validate_host(h, "tw_skip_score_assignments", true, true);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  // 128-in-span tiles, a service's tiles consecutive: [tile prob | tile start | first tile of every problem]
  const int P = h->n_problems;
  std::vector<int32_t> tprob, tstart, tile0((size_t)P);
  for (int p = 0; p < P; ++p) {
    tile0[p] = (int32_t)tprob.size();
    const int64_t n = h->prob_in_off[p + 1] - h->prob_in_off[p];
    for (int64_t i0 = 0; i0 < n; i0 += kAssessThreads) {
      tprob.push_back(p);
      tstart.push_back((int32_t)i0);
    }
  }
  const int nt = (int)tprob.size();
  tprob.insert(tprob.end(), tstart.begin(), tstart.end());
  tprob.insert(tprob.end(), tile0.begin(), tile0.end());
  CU(eng->skip_tiles.reserve(tprob.size()));
  CU(eng->skip_tile_sum.reserve((size_t)nt));
  CU(eng->skip_tile_cnt.reserve((size_t)nt * TW_SKIP_ASSESS_NCODES));
  CU(cudaMemcpyAsync(eng->skip_tiles.p, tprob.data(), tprob.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  AssessOut ao{score_out, code_out, margin_out, prob_sum_out, prob_count_out};
  CU(launch_skip_assess(*dev, *sd, assign, top2, ao, eng->skip_tiles.p, eng->skip_tiles.p + nt, nt,
                        eng->skip_tiles.p + 2 * nt, eng->skip_tile_sum.p, eng->skip_tile_cnt.p, s, eng->launches));
  CU(cudaStreamSynchronize(s));    // the tile lists go out of scope
  return TW_OK;
}

int tw_build_dist_samples(tw_engine* eng, int32_t n, const int64_t* start, const int64_t* end, const int8_t* label,
                          int32_t E, int64_t large_delay, int32_t* key_out, int64_t* val_out, void* stream_) {
  if (!eng || n < 0 || !start || !end || !label || !key_out || !val_out || E < 1 || E > TW_MAX_E)
    return fail(TW_ERR_INVALID, "tw_build_dist_samples: bad argument");
  CU(cudaSetDevice(eng->device));
  CU(launch_build_dist(n, start, end, label, E, large_delay, key_out, val_out, (cudaStream_t)stream_, eng->launches));
  return TW_OK;
}

int tw_gmm_work(tw_engine* eng, uint64_t* em_evals_out, int reset) {
  if (!eng || !em_evals_out) return fail(TW_ERR_INVALID, "tw_gmm_work: NULL argument");
  CU(cudaSetDevice(eng->device));
  CU(cudaDeviceSynchronize());
  unsigned long long v = 0;
  CU(gmm_work_read(&v, reset != 0));
  *em_evals_out = v;
  return TW_OK;
}

int tw_measure_fp64_peak(tw_engine* eng, double* tflops_out, void* stream_) {
  if (!eng || !tflops_out) return fail(TW_ERR_INVALID, "tw_measure_fp64_peak: NULL argument");
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  CU(eng->fp64_sink.reserve(1));
  double* sink = eng->fp64_sink.p;
  const int blocks = eng->n_sm * 8, iters = 1 << 15;
  cudaEvent_t a, b;
  CU(cudaEventCreate(&a));
  CU(cudaEventCreate(&b));
  CU(launch_fp64_peak(blocks, 1 << 10, sink, s, eng->launches));   // warm-up
  double best = 0.0;
  for (int rep = 0; rep < 3; ++rep) {
    CU(cudaEventRecord(a, s));
    CU(launch_fp64_peak(blocks, iters, sink, s, eng->launches));
    CU(cudaEventRecord(b, s));
    CU(cudaEventSynchronize(b));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, a, b));
    const double flops = 2.0 * 8.0 * (double)iters * 256.0 * (double)blocks;
    const double tf = flops / (ms * 1e-3) / 1e12;
    if (tf > best) best = tf;
  }
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  *tflops_out = best;
  return TW_OK;
}

int tw_ground_truth(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const tw_trace_keys* keys,
                    const int32_t* host_trace_n, int32_t* truth_out, void* stream_) {
  if (!eng || !dev || !keys || !host_trace_n || !truth_out) return fail(TW_ERR_INVALID, "tw_ground_truth: NULL argument");
  int rc = validate_host(h, "tw_ground_truth", false, false);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  const int P = h->n_problems;
  std::vector<int64_t> tab_off((size_t)P + 1, 0);
  for (int p = 0; p < P; ++p) {
    if (host_trace_n[p] < 0) return fail(TW_ERR_INVALID, "tw_ground_truth: negative trace range");
    tab_off[p + 1] = tab_off[p] + (int64_t)(h->prob_ep_off[p + 1] - h->prob_ep_off[p]) * host_trace_n[p];
  }
  if (tab_off[P] > (int64_t)1 << 32) return fail(TW_ERR_RANGE_LIMIT, "tw_ground_truth: trace numbers of a service are too sparse");
  CU(eng->truth_tab.reserve((size_t)tab_off[P]));
  CU(eng->truth_tab_off.reserve((size_t)P + 1));
  CU(eng->in_prob.reserve((size_t)h->n_in_total));
  CU(cudaMemcpyAsync(eng->truth_tab_off.p, tab_off.data(), tab_off.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  CU(launch_in_prob(*dev, eng->in_prob.p, s, eng->launches));
  CU(launch_ground_truth(*dev, keys->in_trace, keys->out_trace, keys->prob_trace_lo, keys->prob_trace_n,
                         eng->truth_tab_off.p, tab_off[P], eng->truth_tab.p, eng->in_prob.p, truth_out, s, eng->launches));
  CU(cudaStreamSynchronize(s));    // tab_off goes out of scope
  return TW_OK;
}

int tw_find_order(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const int32_t* truth, uint32_t* violated_out,
                  void* stream_) {
  if (!eng || !dev || !truth || !violated_out) return fail(TW_ERR_INVALID, "tw_find_order: NULL argument");
  int rc = validate_host(h, "tw_find_order", false, false);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  CU(eng->in_prob.reserve((size_t)h->n_in_total));
  CU(eng->order_missing.reserve(1));
  CU(launch_in_prob(*dev, eng->in_prob.p, s, eng->launches));
  CU(launch_find_order(*dev, truth, eng->in_prob.p, violated_out, eng->order_missing.p, s, eng->launches));
  int missing = 0;
  CU(cudaMemcpyAsync(&missing, eng->order_missing.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (missing) return fail(TW_ERR_INVALID, "tw_find_order: an incoming span has no child at some callee%s", "");
  return TW_OK;
}

int tw_accuracy(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const int32_t* truth, const int32_t* assign,
                const int32_t* topk_idx, const uint8_t* topk_cnt, const int32_t* in_trace, int32_t n_traces,
                const uint8_t* prob_first, uint64_t* per_prob_out, uint64_t* e2e_out, void* stream_) {
  if (!eng || !dev || !truth || !assign || !per_prob_out || !e2e_out) return fail(TW_ERR_INVALID, "tw_accuracy: NULL argument");
  if ((topk_idx != nullptr) != (topk_cnt != nullptr)) return fail(TW_ERR_INVALID, "tw_accuracy: topk_idx and topk_cnt go together");
  int rc = validate_host(h, "tw_accuracy", false, false);
  if (rc) return rc;
  if (n_traces < 0 || !in_trace) n_traces = 0;
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  CU(eng->in_prob.reserve((size_t)h->n_in_total));
  CU(eng->acc_flags.reserve((size_t)3 * (size_t)n_traces + 8));
  CU(eng->acc_first.reserve((size_t)n_traces + 1));
  CU(cudaMemsetAsync(eng->acc_flags.p, 0, (size_t)3 * (size_t)n_traces + 1, s));
  CU(cudaMemsetAsync(eng->acc_first.p, 0, ((size_t)n_traces + 1) * sizeof(unsigned long long), s));
  CU(cudaMemsetAsync(per_prob_out, 0, (size_t)h->n_problems * 2 * sizeof(uint64_t), s));
  CU(cudaMemsetAsync(e2e_out, 0, 4 * sizeof(uint64_t), s));
  CU(launch_in_prob(*dev, eng->in_prob.p, s, eng->launches));
  CU(launch_accuracy(*dev, truth, assign, topk_idx, topk_cnt, n_traces ? in_trace : nullptr, eng->in_prob.p, prob_first,
                     n_traces, (unsigned long long*)per_prob_out, eng->acc_flags.p, eng->acc_first.p,
                     (unsigned long long*)e2e_out, s, eng->launches));
  return TW_OK;
}

// The host checks of tw_assemble_traces: the offset tables and int32 node ids.
static int trace_check(const tw_batch* h, const char* who) {
  int rc = validate_host(h, who, false, true);
  if (rc) return rc;
  const int64_t n_nodes = h->n_in_total + h->n_out_total;
  if (n_nodes >= ((int64_t)1 << 31))
    return fail(TW_ERR_RANGE_LIMIT, (std::string(who) + ": %s nodes do not fit int32 node ids").c_str(),
                std::to_string(n_nodes).c_str());
  return TW_OK;
}

// The join of tw_assemble_traces after trace_check: its launches, the read-back of its error words and
// round flags, and its errors (named after `who`).  A NULL parent_out / size_out goes to the engine's
// eng->trace_parent / eng->trace_size.  Leaves the caller-claim words in eng->trace_claim.
static int trace_join(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const int32_t* assign,
                      const int32_t* in_caller, int32_t* parent_out, int32_t* root_out, int32_t* size_out,
                      const char* who, cudaStream_t s) {
  const int64_t n_in = h->n_in_total, n_out = h->n_out_total, n_nodes = n_in + n_out;
  const int rounds = trace_rounds(n_nodes);
  if (!parent_out) {
    CU(eng->trace_parent.reserve((size_t)n_nodes));
    parent_out = eng->trace_parent.p;
  }
  if (!size_out) {
    CU(eng->trace_size.reserve((size_t)n_nodes));
    size_out = eng->trace_size.p;
  }
  CU(eng->trace_claim.reserve((size_t)n_out));
  CU(eng->trace_flags.reserve((size_t)(4 + rounds)));
  int32_t* err = eng->trace_flags.p;
  int* changed = (int*)(eng->trace_flags.p + 4);
  CU(launch_assemble_traces(*dev, h->prob_tuple_off[h->n_problems], assign, in_caller, parent_out, root_out, size_out,
                            eng->trace_claim.p, err, changed, rounds, eng->n_sm, s, eng->launches));
  std::vector<int32_t> flags((size_t)(4 + rounds));
  CU(cudaMemcpyAsync(flags.data(), err, flags.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  eng->trace_rounds_launched = rounds;
  eng->trace_rounds_run = 1;                               // round r > 0 runs iff round r - 1 moved a node
  while (eng->trace_rounds_run < rounds && flags[4 + eng->trace_rounds_run - 1]) ++eng->trace_rounds_run;
  eng->trace_still = 0;                                    // the first round that moved no node (rounds: none)
  while (eng->trace_still < rounds && flags[4 + eng->trace_still]) ++eng->trace_still;
  const int32_t none = 0x7f7f7f7f;
  const char* what[4] = {"out-span node %s is the child of two in-spans%s",
                         "out-span node %s is the caller of two in-spans%s",
                         "in-span node %s has a child index outside its callee's list%s",
                         "in-span node %s has a caller that is not an out-span node%s"};
  for (int k : {3, 1, 2, 0})                               // the callers first, as traces.parents_host
    if (flags[k] != none) {
      const std::string msg = std::string(who) + ": " + what[k];
      return fail(TW_ERR_INVALID, msg.c_str(), std::to_string(flags[k]).c_str(), "");
    }
  return TW_OK;
}

int tw_assemble_traces(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const int32_t* assign,
                       const int32_t* in_caller, int32_t* parent_out, int32_t* root_out, int32_t* size_out,
                       void* stream_) {
  if (!eng || !dev || !assign || !in_caller || !parent_out || !root_out || !size_out)
    return fail(TW_ERR_INVALID, "tw_assemble_traces: NULL argument");
  int rc = trace_check(h, "tw_assemble_traces");
  if (rc) return rc;
  CU(cudaSetDevice(eng->device));
  return trace_join(eng, dev, h, assign, in_caller, parent_out, root_out, size_out, "tw_assemble_traces",
                    (cudaStream_t)stream_);
}

int tw_critical_paths(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const tw_times_f64* f64,
                      const int32_t* assign, const int32_t* in_caller, double slow_us, const tw_critical_out* out,
                      void* stream_) {
  if (!eng || !dev || !assign || !in_caller || !out || !out->root || !out->on_path || !out->self_us ||
      !out->culprit || !out->server_us || !out->server_visits || !out->call_us || !out->requests ||
      (f64 ? (!f64->in_start || !f64->in_end || !f64->out_start || !f64->out_end)
           : (!dev->in_start || !dev->in_end || !dev->out_start || !dev->out_end)))
    return fail(TW_ERR_INVALID, "tw_critical_paths: NULL argument");
  int rc = trace_check(h, "tw_critical_paths");
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  const int64_t n_in = h->n_in_total;
  CU(eng->cp_level.reserve((size_t)n_in));
  CU(eng->cp_wlo.reserve((size_t)n_in));
  CU(eng->cp_whi.reserve((size_t)n_in));
  CU(eng->cp_slow.reserve((size_t)n_in));
  CU(eng->cp_cmax.reserve((size_t)n_in));
  CU(eng->cp_act.reserve((size_t)kCpMaxLevels));
  rc = trace_join(eng, dev, h, assign, in_caller, nullptr, out->root, nullptr, "tw_critical_paths", s);
  if (rc) return rc;
  // Depth of the trees from the rounds: when round k moved no node, every node had reached its root in
  // rounds 0 .. k - 1, which climb 2^k links (none when k = 0); an in-span at depth 2m links is walked at
  // level m.  When every round moved a node (a cycle of links can keep moving), or the bound exceeds
  // kCpMaxLevels: kCpMaxLevels.  Rounds run in place, so a node can climb further than 2^k links in them
  // and the count depends on the order threads ran in; the last level walks whatever lies deeper itself,
  // so only the launch count does, not the results.
  int levels = kCpMaxLevels;
  const int k = eng->trace_still;
  if (k < eng->trace_rounds_launched && (k == 0 ? 1 : ((int64_t)1 << k) / 2 + 1) < kCpMaxLevels)
    levels = k == 0 ? 1 : (int)(((int64_t)1 << k) / 2 + 1);
  if (eng->cp_force_levels) levels = eng->cp_force_levels;
  eng->cp_levels = levels;
  CpScratch sc{eng->cp_level.p, eng->cp_wlo.p, eng->cp_whi.p, eng->cp_slow.p, eng->cp_cmax.p, eng->cp_act.p};
  CU(launch_critical_paths(*dev, f64, assign, eng->trace_claim.p, eng->trace_parent.p, slow_us, *out, sc, levels,
                           eng->n_sm, s, eng->launches));
  return TW_OK;
}

int tw_request_confidence(tw_engine* eng, const tw_batch* dev, const tw_batch* h, const int32_t* assign,
                          const int32_t* in_caller, const double* score, const uint8_t* code,
                          const tw_score_out* top, const tw_confidence_out* out, void* stream_) {
  if (!eng || !dev || !assign || !in_caller || !score || !code || !top || !top->topk_score || !top->topk_idx ||
      !top->topk_cnt || !out || !out->root || !out->p || !out->ell || !out->decisions || !out->zero ||
      !out->log_conf || !out->conf || !out->weakest || !out->weakest_p || !out->est_accuracy || !out->requests ||
      !out->expected_exact)
    return fail(TW_ERR_INVALID, "tw_request_confidence: NULL argument");
  int rc = trace_check(h, "tw_request_confidence");
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream_;
  CU(cudaSetDevice(eng->device));
  const int64_t n_in = h->n_in_total;
  CU(eng->cf_wbits.reserve((size_t)n_in));
  CU(eng->cf_seg_conf.reserve((size_t)h->n_problems));
  CU(eng->cf_seg_req.reserve((size_t)h->n_problems));
  CU(eng->cf_flag.reserve(1));
  rc = trace_join(eng, dev, h, assign, in_caller, nullptr, out->root, nullptr, "tw_request_confidence", s);
  if (rc) return rc;
  CfScratch sc{eng->cf_wbits.p, eng->cf_seg_conf.p, eng->cf_seg_req.p, eng->cf_flag.p};
  CU(launch_request_confidence(*dev, assign, score, code, *top, *out, sc, eng->n_sm, s, eng->launches));
  int32_t big = 0;
  CU(cudaMemcpyAsync(&big, eng->cf_flag.p, sizeof big, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (big != 0x7f7f7f7f)
    return fail(TW_ERR_RANGE_LIMIT, "tw_request_confidence: the request rooted at in-span node %s has 2^21 or more "
                "decisions (its fixed-point sum could overflow)", std::to_string(big).c_str());
  return TW_OK;
}

// Test hook, not part of the ABI header: later tw_critical_paths calls launch `levels` levels (1 ..
// kCpMaxLevels), or as many as the join's rounds give (0).
int tw_debug_critical_force_levels(tw_engine* eng, int levels) {
  if (!eng) return fail(TW_ERR_INVALID, "tw_debug_critical_force_levels: NULL engine");
  if (levels < 0 || levels > kCpMaxLevels)
    return fail(TW_ERR_INVALID, "tw_debug_critical_force_levels: %s levels (0 .. 64)", std::to_string(levels).c_str());
  eng->cp_force_levels = levels;
  return TW_OK;
}

// Test hook, not part of the ABI header: the level launches of the last tw_critical_paths.
int tw_debug_critical_levels(tw_engine* eng, int* levels) {
  if (!eng || !levels) return fail(TW_ERR_INVALID, "tw_debug_critical_levels: NULL argument");
  *levels = eng->cp_levels;
  return TW_OK;
}

// Test hook, not part of the ABI header: pointer-jumping rounds the last tw_assemble_traces launched and
// the rounds of them that ran (the others returned at once after a round that moved no node).
int tw_debug_trace_rounds(tw_engine* eng, int* launched, int* run) {
  if (!eng || !launched || !run) return fail(TW_ERR_INVALID, "tw_debug_trace_rounds: NULL argument");
  *launched = eng->trace_rounds_launched;
  *run = eng->trace_rounds_run;
  return TW_OK;
}

static int need_bound(tw_engine* eng, const char* who) {
  if (!eng || !eng->bound) return fail(TW_ERR_INVALID, "%s: no batch bound", who);
  cudaError_t e = cudaSetDevice(eng->device);
  if (e != cudaSuccess) return fail(TW_ERR_CUDA, "%s: %s", who, cudaGetErrorString(e));
  return TW_OK;
}

int tw_params_pass0(tw_engine* eng, const int64_t* prob_gauss_off, double* gauss_out, void* stream) {
  int rc = need_bound(eng, "tw_params_pass0");
  if (rc) return rc;
  CU(launch_params0(eng->dev, eng->in_end_sorted.p, eng->out_end_sorted.p, prob_gauss_off, eng->batch_prob.p,
                    eng->batch_idx.p, eng->n_batches_total, gauss_out, eng->shifted ? eng->prob_shift.p : nullptr,
                    (cudaStream_t)stream, eng->launches));
  return TW_OK;
}

int tw_score_topk(tw_engine* eng, const tw_params* params, const tw_score_out* out, void* stream) {
  int rc = need_bound(eng, "tw_score_topk");
  if (rc) return rc;
  if (!out || !out->cut || !out->n_feasible) return fail(TW_ERR_INVALID, "tw_score_topk: cut and n_feasible are required");
  if (params && (!out->topk_score || !out->topk_idx || !out->topk_cnt))
    return fail(TW_ERR_INVALID, "tw_score_topk: params given but topk outputs missing");
  if ((out->used_lo != nullptr) != (out->used_bits != nullptr) || (out->used_lo != nullptr) != (out->used_wide != nullptr))
    return fail(TW_ERR_INVALID, "tw_score_topk: used_lo / used_bits / used_wide go together");
  const int keep = (out->flags & TW_SCORE_KEEP_WINDOWS) != 0;
  if (keep && !eng->windows_valid)
    return fail(TW_ERR_INVALID, "tw_score_topk: TW_SCORE_KEEP_WINDOWS before any full call on this batch");
  if (keep && !params) return TW_OK;   // nothing to do
  cudaStream_t s = (cudaStream_t)stream;
  tw_score_out o = *out;
  if (!o.used_lo) {                    // the perfect-cut pass reads the maps: keep them in engine scratch
    const size_t nt = (size_t)eng->dev_n_tuple;
    CU(eng->own_used_lo.reserve(nt));
    CU(eng->own_used_bits.reserve(2 * nt));
    CU(eng->own_used_wide.reserve((size_t)eng->dev.n_in_total));
    o.used_lo = eng->own_used_lo.p;
    o.used_bits = eng->own_used_bits.p;
    o.used_wide = eng->own_used_wide.p;
  }
  tw_params sp;
  if (params) {
    rc = scoring_params(eng, params, sp, s);
    if (rc) return rc;
    params = &sp;
  }
  ScoreTiles st;
  st.tile_prob = eng->score_tiles.p;
  st.tile_start = eng->score_tiles.p + eng->n_tiles;
  st.tile_win = eng->tile_win.p;
  st.overflow = eng->tile_overflow.p;
  st.n_tiles = eng->n_tiles;
  for (int q = 0; q <= TW_MAX_E; ++q) st.class_off[q] = eng->class_off[q];
  TileList wide{eng->wide_tiles.p, eng->wide_tiles.p + eng->n_wide, eng->n_wide, kWideThreads - 1,
                eng->wide_tiles.p + 3 * eng->n_wide};
  // work-balanced scoring kernel (one launch per E present); flagged tiles are redone by the
  // sequential kernel; PerfectCut flags from the candidate maps
  CU(launch_score3(eng->dev, params, o, keep, st, eng->prev_idx.p, s, eng->launches));
  CU(launch_score_redo(eng->dev, params, o, wide, eng->prev_idx.p, eng->tile_overflow.p, eng->n_sm, eng->err_flag.p, s,
                       eng->launches));
  if (!keep) {
    CU(launch_cut(eng->dev, o, st, eng->prev_idx.p, s, eng->launches));
    eng->windows_valid = true;
  }
  return TW_OK;
}

int tw_stitch(tw_engine* eng, const tw_params* params, const uint8_t* cut, const tw_score_out* undeleted,
              const tw_pass_out* out, void* stream) {
  int rc = need_bound(eng, "tw_stitch");
  if (rc) return rc;
  if (!params || !cut || !out || !out->assign || !out->mis_rank || !out->n_cand)
    return fail(TW_ERR_INVALID, "tw_stitch: params, cut, assign, mis_rank, n_cand are required");
  if (out->topk_score && (!out->topk_idx || !out->topk_cnt)) return fail(TW_ERR_INVALID, "tw_stitch: partial topk outputs");
  tw_score_out spec;
  memset(&spec, 0, sizeof spec);
  if (undeleted) {
    if (!undeleted->topk_score || !undeleted->topk_idx || !undeleted->topk_cnt || !undeleted->n_feasible ||
        !undeleted->used_lo || !undeleted->used_bits || !undeleted->used_wide)
      return fail(TW_ERR_INVALID, "tw_stitch: `undeleted` needs top-K, n_feasible and the used maps");
    spec = *undeleted;
  }
  tw_params sp;
  rc = scoring_params(eng, params, sp, (cudaStream_t)stream);
  if (rc) return rc;
  StitchUnits ub{eng->unit_prob.p, eng->unit_lo.p, eng->unit_hi.p, eng->unit_count.p, eng->unit_count.p + 1};
  CU(launch_stitch(eng->dev, sp, cut, spec, *out, eng->taken.p, eng->taken_words, eng->node_limit, ub,
                   eng->unit_min, eng->stitch_blocks, eng->stitch_layout, eng->stitch_tables.p, eng->err_flag.p,
                   (cudaStream_t)stream, eng->launches));
  return TW_OK;
}

// Test hook, not part of the ABI header: run the stitch of the bound batch on `blocks` blocks (1 ..
// the grid the bind sized), so that one warp takes many units; blocks <= 0 restores the bind's grid.
// Returns the grid now in effect, or TW_ERR_INVALID.
int tw_debug_stitch_grid(tw_engine* eng, int blocks) {
  int rc = need_bound(eng, "tw_debug_stitch_grid");
  if (rc) return rc;
  if (blocks > eng->stitch_blocks_max) return fail(TW_ERR_INVALID, "tw_debug_stitch_grid: more blocks than the bind sized");
  eng->stitch_blocks = blocks > 0 ? blocks : eng->stitch_blocks_max;
  return eng->stitch_blocks;
}

int tw_score_assignments(tw_engine* eng, const tw_params* params, const int32_t* assign, const tw_score_out* final_topk,
                         double* score_out, uint8_t* code_out, double* margin_out, double* prob_sum_out,
                         int32_t* prob_count_out, void* stream) {
  int rc = need_bound(eng, "tw_score_assignments");
  if (rc) return rc;
  if (!params || !assign || !score_out || !code_out || !prob_sum_out || !prob_count_out)
    return fail(TW_ERR_INVALID, "tw_score_assignments: params, assign, score, code and the per-service outputs are required");
  if ((final_topk != nullptr) != (margin_out != nullptr))
    return fail(TW_ERR_INVALID, "tw_score_assignments: final_topk and margin_out go together");
  if (final_topk && (!final_topk->topk_score || !final_topk->topk_idx || !final_topk->topk_cnt))
    return fail(TW_ERR_INVALID, "tw_score_assignments: final_topk needs topk_score, topk_idx and topk_cnt");
  if (params->mode == TW_PARAMS_GAUSS_BATCHED ? (!params->prob_gauss_off || !params->gauss)
                                              : (params->mode != TW_PARAMS_MIXTURE || !params->mix))
    return fail(TW_ERR_INVALID, "tw_score_assignments: bad params");
  cudaStream_t s = (cudaStream_t)stream;
  const int P = eng->dev.n_problems;
  if (!eng->prob_tile0_uploaded) {
    CU(eng->assess_tile0.reserve((size_t)P));
    CU(cudaMemcpyAsync(eng->assess_tile0.p, eng->prob_tile0.data(), (size_t)P * sizeof(int32_t),
                       cudaMemcpyHostToDevice, s));
    eng->prob_tile0_uploaded = true;
  }
  CU(eng->assess_tile_sum.reserve((size_t)eng->n_tiles));
  CU(eng->assess_tile_cnt.reserve((size_t)eng->n_tiles * TW_ASSESS_NCODES));
  tw_params sp;
  rc = scoring_params(eng, params, sp, s);
  if (rc) return rc;
  AssessOut ao{score_out, code_out, margin_out, prob_sum_out, prob_count_out};
  CU(launch_assess(eng->dev, sp, assign, final_topk, ao, eng->score_tiles.p, eng->score_tiles.p + eng->n_tiles,
                   eng->n_tiles, eng->assess_tile0.p, eng->assess_tile_sum.p, eng->assess_tile_cnt.p, s,
                   eng->launches));
  return TW_OK;
}

int tw_delays(tw_engine* eng, const int32_t* assign, const int64_t* term_sample_off, double* delays,
              int32_t* counts, void* stream) {
  int rc = need_bound(eng, "tw_delays");
  if (rc) return rc;
  CU(launch_delays(eng->dev, assign, term_sample_off, eng->term_ep.p, eng->ep_prob.p, delays, counts,
                   eng->shifted ? eng->prob_shift.p : nullptr, (cudaStream_t)stream, eng->launches));
  return TW_OK;
}

// NumPy legacy RandomState(seed).random_sample() stream (MT19937; std::mt19937 has the same
// init_genrand seeding and tempering): (a >> 5, b >> 6) -> (a * 2^26 + b) / 2^53.
static void numpy_random_samples(uint32_t seed, int count, std::vector<double>& out) {
  std::mt19937 mt(seed);
  out.resize(count);
  for (int i = 0; i < count; ++i) {
    uint32_t a = (uint32_t)mt() >> 5, b = (uint32_t)mt() >> 6;
    out[i] = (a * 67108864.0 + b) / 9007199254740992.0;
  }
}

static int gmm_prepare(tw_engine* eng, uint32_t seed_select, cudaStream_t s) {
  const int nt = eng->dev.n_term_total;
  CU(eng->gmm_max_n.reserve((size_t)nt));
  CU(eng->gmm_mean_var.reserve((size_t)nt * 2));
  CU(eng->gmm_skip.reserve((size_t)nt + 64));   // + histogram / cursors of the final-fit grouping
  CU(eng->gmm_bic.reserve((size_t)nt * TW_GMM_MAX_COMP));
  CU(eng->gmm_cen.reserve((size_t)nt * TW_GMM_MAX_COMP * TW_GMM_MAX_COMP));   // one slab per K
  if (!eng->gmm_fork.ready) {
    CU(cudaEventCreateWithFlags(&eng->gmm_fork.fork, cudaEventDisableTiming));
    for (int q = 0; q < TW_GMM_MAX_COMP; ++q) {
      CU(cudaStreamCreateWithFlags(&eng->gmm_fork.side[q], cudaStreamNonBlocking));
      CU(cudaEventCreateWithFlags(&eng->gmm_fork.join[q], cudaEventDisableTiming));
    }
    eng->gmm_fork.ready = true;
  }
  CU(eng->gmm_stream.reserve((size_t)tw_engine::kStreamLen, &eng->gmm_seed_valid));
  CU(eng->gmm_stream100.reserve(16, &eng->gmm_stream100_valid));
  if (!eng->gmm_stream100_valid) {
    std::vector<double> s100;
    numpy_random_samples(100u, 16, s100);
    CU(cudaMemcpyAsync(eng->gmm_stream100.p, s100.data(), 16 * sizeof(double), cudaMemcpyHostToDevice, s));
    CU(cudaStreamSynchronize(s));
    eng->gmm_stream100_valid = true;
  }
  if (!eng->gmm_seed_valid || eng->gmm_seed != seed_select) {
    std::vector<double> st;
    numpy_random_samples(seed_select, tw_engine::kStreamLen, st);
    CU(cudaMemcpyAsync(eng->gmm_stream.p, st.data(), st.size() * sizeof(double), cudaMemcpyHostToDevice, s));
    CU(cudaStreamSynchronize(s));
    eng->gmm_seed = seed_select;
    eng->gmm_seed_valid = true;
  }
  return TW_OK;
}

int tw_gmm_refit(tw_engine* eng, const int64_t* term_sample_off, const double* delays, const int32_t* counts,
                 uint32_t seed_select, const uint32_t* prob_base_skip, const int32_t* term_order,
                 double* mix_out, int32_t* n_selected_out, void* stream) {
  int rc = need_bound(eng, "tw_gmm_refit");
  if (rc) return rc;
  if (!term_sample_off || !delays || !counts || !mix_out) return fail(TW_ERR_INVALID, "tw_gmm_refit: NULL argument");
  cudaStream_t s = (cudaStream_t)stream;
  rc = gmm_prepare(eng, seed_select, s);
  if (rc) return rc;
  const int nt = eng->dev.n_term_total;
  CU(launch_gmm_prep(nt, term_sample_off, delays, counts, eng->gmm_max_n.p, eng->gmm_mean_var.p, s, eng->launches));
  CU(launch_gmm_skip(eng->dev.n_problems, eng->dev.prob_ep_off, eng->dev.ep_term_off, term_order, eng->gmm_max_n.p,
                     prob_base_skip, eng->gmm_skip.p, s, eng->launches));
  CU(launch_gmm_fit(nt, term_sample_off, delays, counts, eng->gmm_max_n.p, eng->gmm_mean_var.p, eng->gmm_skip.p,
                    eng->gmm_stream.p, tw_engine::kStreamLen, eng->gmm_stream100.p, eng->gmm_bic.p, eng->gmm_cen.p,
                    mix_out, n_selected_out, eng->err_flag.p, &eng->gmm_fork, s, eng->launches));
  return TW_OK;
}

int tw_gmm_stream_draws(tw_engine* eng, const int64_t* term_sample_off, const double* delays,
                        const int32_t* counts, uint32_t* prob_draws_out, void* stream) {
  int rc = need_bound(eng, "tw_gmm_stream_draws");
  if (rc) return rc;
  if (!term_sample_off || !delays || !counts || !prob_draws_out)
    return fail(TW_ERR_INVALID, "tw_gmm_stream_draws: NULL argument");
  cudaStream_t s = (cudaStream_t)stream;
  rc = gmm_prepare(eng, eng->gmm_seed_valid ? eng->gmm_seed : 10u, s);
  if (rc) return rc;
  const int nt = eng->dev.n_term_total;
  CU(launch_gmm_prep(nt, term_sample_off, delays, counts, eng->gmm_max_n.p, eng->gmm_mean_var.p, s, eng->launches));
  CU(launch_gmm_draws(eng->dev.n_problems, eng->dev.prob_ep_off, eng->dev.ep_term_off, eng->gmm_max_n.p,
                      prob_draws_out, s, eng->launches));
  return TW_OK;
}

}  // extern "C"
