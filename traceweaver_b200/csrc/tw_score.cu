// tw_score.cu — the prev-index scan, and the sequential redo of the scoring tiles that the
// work-balanced kernel (tw_score3.cu) flags: candidate ranges wider than its 64-bit maps, more
// combinations than it takes, staging overflow, equal scores or NaN.  The redo enumerates in the
// reference's own order and tie rule: candidate enumeration + likelihood scoring + top-K on the
// undeleted lists, the candidate maps and the perfect-cut flags of the flagged tiles.
//
// Replaces (reference: .../algorithms/traceweaver_v3.py = V3, traceweaver_v1.py = V1)
//   FindTopKAssignments(K=5, out_span_partitions)   V3:1185  (DfsTraverseX V3:292-351,
//       ScoreAssignmentAsPerInvocationGraph V1:259-361, GetEpPairCost V1:117-139)
//   CreateWindows2 pre-processing + PerfectCut       V3:1020-1051
//
// Mapping to the machine: a one-warp CTA owns a wide tile of kWideThreads - 1 consecutive in-spans
// of one service (in-spans are sorted by start), one lane per in-span.  Because both sides are
// sorted by start, all candidates of the tile lie in one contiguous slice of each ep's out list: the
// slice's start/end timestamps are staged once into shared memory (read in place when the slice is
// too large) and every search step then runs out of shared memory.  Likelihood parameters of the
// tile's 100-span batches are staged alongside.  The last lane enumerates the tile's carry-in "prev"
// in-span (the latest-ending in-span before the tile) so that PerfectCut(i) = disjoint(cand(prev(i)),
// cand(i)) is resolved inside the CTA from candidate maps of 32 * kWideW bits per ep in shared
// memory.  The top-K search is warp_topk_search below.
#include "tw_kernels.cuh"

namespace tw {

// ---------------------------------------------------------------------------------------------
// prev_index(i) = arg max_{j < i} in_end[j], ties to the later j   (V3:1026-1032)
// one warp per problem, shuffle scan
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_prev_index(tw_batch b, int32_t* __restrict__ prev_idx) {
  int warp = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  int lane = threadIdx.x & 31;
  if (warp >= b.n_problems) return;
  int64_t off = b.prob_in_off[warp];
  int n = (int)(b.prob_in_off[warp + 1] - off);
  const int64_t* ie = b.in_end + off;
  int64_t cmax = INT64_MIN;
  int cidx = 0;
  for (int base = 0; base < n; base += 32) {
    int i = base + lane;
    int64_t v = i < n ? ie[i] : INT64_MIN;
    int vi = i;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int64_t ov = __shfl_up_sync(0xffffffffu, v, d);
      int oi = __shfl_up_sync(0xffffffffu, vi, d);
      if (lane >= d && !(v >= ov)) { v = ov; vi = oi; }
    }
    if (!(v >= cmax)) { v = cmax; vi = cidx; }   // fold the carry (earlier elements)
    int64_t pv = __shfl_up_sync(0xffffffffu, v, 1);
    int pi = __shfl_up_sync(0xffffffffu, vi, 1);
    if (lane == 0) { pv = cmax; pi = cidx; }
    (void)pv;
    if (i < n) prev_idx[off + i] = i == 0 ? 0 : pi;
    cmax = __shfl_sync(0xffffffffu, v, 31);
    cidx = __shfl_sync(0xffffffffu, vi, 31);
  }
}

cudaError_t launch_prev_index(const tw_batch& b, int32_t* prev_idx, cudaStream_t s, int64_t& launches) {
  int warps_per_block = 4;
  int blocks = (b.n_problems + warps_per_block - 1) / warps_per_block;
  k_prev_index<<<blocks, warps_per_block * 32, 0, s>>>(b, prev_idx);
  return after_launch(launches);
}

// ---------------------------------------------------------------------------------------------
// warp-level top-K search (the search tier of k_stitch, stitch_search_lanes, runs the same steps in
// its own copy: any change to that out-of-line function moves ptxas's register allocation of the
// stitch's hot loop around the call, which cost 0.5 ms per hotel step on an H100 80GB at 400 W)
// ---------------------------------------------------------------------------------------------
// Every lane with `pending` set finds the top-K tuples of its in-span i = [in_s, in_e] among the
// candidates `taken` does not exclude, and hands the sorted list and its leaf count to
// publish(tk, leaves) on its own lane.  All 32 lanes call this converged.  `w` (one window per ep) is
// the same on every lane; lo[e] is the lane's first candidate in w[e].  `tbl` / `sid` is a slab of
// kCap term-table slots.  params(bq) returns the likelihood parameters of 100-span batch batch0 + bq,
// where batch0 is the tile's or window's first batch: the batch bits of a slot id and the lazy path's
// batch count from there.
// mark(owner, c, lo_abs, coop) sees every feasible tuple c of lane `owner`'s in-span (lo_abs = the
// owner's first candidate per ep, original index); with coop set, several lanes mark the same owner.
//
// 1. Heavy in-spans (more than kCoopCombos candidate combinations, tables within the slab), one at a
//    time by the whole warp.  A lane that walks thousands of tuples alone keeps one lane of 32 busy;
//    here the owner lays out its term tables, all lanes evaluate the slots, then take the
//    combinations lane, lane + 32, ... (ascending combination index = depth-first leaf order), keep
//    their own top K, and the warp merges the heads.  If two of the six best scores are equal, or a
//    score is NaN, only the literal heapq replay of topk_offer reproduces the reference's order: the
//    in-span stays pending and its owner redoes it alone in step 2.
// 2. Rounds: the pending lanes' tables are laid out back to back in the slab (exclusive prefix sum of
//    their sizes), all lanes evaluate the slots, then each lane walks its own tuples.  A lane whose
//    tables do not fit even an empty slab scores every leaf from scratch (lazy path).
// Leaf counts of step 2 saturate at 0x7fffffff; step 1 only takes fewer than 2^31 combinations.
template <int kCap, int kCoopCombos, class Params, class Taken, class Mark, class Publish>
__device__ __forceinline__ void warp_topk_search(const ProbView& v, const OutWin* w, Params params,
                                                 int batch0, double* tbl, uint8_t* sid, int lane, int i,
                                                 int64_t in_s, int64_t in_e, const int* lo, bool pending,
                                                 Taken taken, Mark mark, Publish publish) {
  const unsigned kAll = 0xffffffffu;
  const int E = v.E;
  int r[TW_MAX_E], lo_abs[TW_MAX_E];
  int tsize = 0;
  if (pending) {
    for (int e = 0; e < E; ++e) {
      lo_abs[e] = w[e].base + lo[e];
      r[e] = range_len(w[e], lo[e], in_e);
    }
    tsize = term_table_size(v, r);
  }
  const int brel = i / TW_PARAM_BATCH - batch0;
  auto eval_slots = [&](int total) {   // GetEpPairCost (V1:117-139) for every slot, all lanes busy
    for (int s = lane; s < total; s += 32) {
      const uint8_t id = sid[s];
      if (id != TW_SLOT_INVALID) tbl[s] = term_logpdf(params(id >> 6), id & 63, tbl[s]);
    }
  };

  // ---- 1. heavy in-spans by the whole warp
  const long long Pown = pending ? combo_count(v, r) : 0;
  unsigned heavy = __ballot_sync(kAll, pending && tsize <= kCap && Pown > kCoopCombos && Pown < (1LL << 31));
  while (heavy) {
    const int L = __ffs(heavy) - 1;
    heavy &= heavy - 1u;
    int lo_b[TW_MAX_E], r_b[TW_MAX_E], o_last_b[TW_MAX_E], lo_abs_b[TW_MAX_E];
    for (int e = 0; e < E; ++e) {
      lo_b[e] = __shfl_sync(kAll, lo[e], L);
      r_b[e] = __shfl_sync(kAll, r[e], L);
      lo_abs_b[e] = w[e].base + lo_b[e];
    }
    const int tsz = __shfl_sync(kAll, tsize, L);
    const long long P_b = __shfl_sync(kAll, Pown, L);
    term_table_last_offsets(v, r_b, o_last_b);
    if (lane == L) term_table_fill(v, in_s, in_e, w, lo, r, o_last_b, brel, taken, tbl, sid);
    __syncwarp();
    eval_slots(tsz);
    __syncwarp();
    TopK part;
    part.clear();
    int leaves = 0;
    bool tie = false;
    enumerate_combos(v, w, lo_b, r_b, o_last_b, sid, lane, 32, P_b,
                     [&](const int* c, const int64_t* ce, long long) {
                       ++leaves;
                       mark(L, c, lo_abs_b, true);
                       const double sc = table_score(v, r_b, lo_abs_b, tbl, c, ce);
                       for (int k = 0; k < part.n; ++k) tie = tie || part.score[k] == sc;
                       tie = tie || sc != sc;
                       topk_offer_sorted(v, part, sc, c);
                     });
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) leaves += __shfl_xor_sync(kAll, leaves, d);
    TopK tkc;
    tkc.clear();
    int head = 0;
    double prev = 0.0;
    for (int round = 0; round <= TW_K; ++round) {
      const double hs = head < part.n ? part.score[head] : -INFINITY;
      double mx = hs;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        const double o = __shfl_xor_sync(kAll, mx, d);
        mx = o > mx ? o : mx;
      }
      if (!(mx > -INFINITY)) break;
      const unsigned who = __ballot_sync(kAll, hs == mx);
      if (__popc(who) > 1 || (round > 0 && mx == prev)) tie = true;
      prev = mx;
      const int wl = __ffs(who) - 1;
      if (round < TW_K) {
        for (int e = 0; e < E; ++e) {
          const int ci = __shfl_sync(kAll, head < part.n ? part.idx[head][e] : -1, wl);
          if (lane == L) tkc.idx[round][e] = ci;
        }
        if (lane == L) { tkc.score[round] = mx; tkc.n = round + 1; }
      }
      if (lane == wl) ++head;
    }
    tie = __any_sync(kAll, tie);
    if (!tie && lane == L) {
      publish(tkc, leaves);
      pending = false;
    }
    __syncwarp();
  }

  // ---- 2. rounds, one lane per in-span
  if (!__any_sync(kAll, pending)) return;
  while (true) {
    int my = pending ? tsize : 0, incl = my;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(kAll, incl, d);
      if (lane >= d) incl += o;
    }
    const int offset = incl - my;
    const bool lazy = pending && offset == 0 && tsize > kCap;
    const bool in_round = pending && !lazy && offset + tsize <= kCap;
    int total = in_round ? offset + tsize : 0;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) total = max(total, __shfl_xor_sync(kAll, total, d));
    int o_last[TW_MAX_E];
    if (in_round) {
      term_table_last_offsets(v, r, o_last);
      term_table_fill(v, in_s, in_e, w, lo, r, o_last, brel, taken, tbl + offset, sid + offset);
    }
    if (lazy) {
      const ParamView pv = params(brel);
      TopK tk;
      tk.clear();
      int leaves = 0;
      enumerate(v, in_s, in_e, w, lo, taken, [&](const int* c, const int64_t* cs, const int64_t* ce) {
        if (leaves < 0x7fffffff) ++leaves;
        mark(lane, c, lo_abs, false);
        topk_offer(v, tk, score_tuple(v, pv, in_s, in_e, cs, ce), c);
      });
      topk_finish(v, tk);
      publish(tk, leaves);
      pending = false;
    }
    __syncwarp();
    eval_slots(total);
    __syncwarp();
    if (in_round) {
      const double* t = tbl + offset;
      const uint8_t* id = sid + offset;
      TopK tk;
      tk.clear();
      int leaves = 0;
      enumerate(v, in_s, in_e, w, lo,
                [&](int e, int o) { return id[o_last[e] + (o - lo_abs[e])] == TW_SLOT_INVALID; },
                [&](const int* c, const int64_t*, const int64_t* ce) {
                  if (leaves < 0x7fffffff) ++leaves;
                  mark(lane, c, lo_abs, false);
                  topk_offer(v, tk, table_score(v, r, lo_abs, t, c, ce), c);
                });
      topk_finish(v, tk);
      publish(tk, leaves);
      pending = false;
    }
    if (!__any_sync(kAll, pending)) break;
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------
// redo kernel
// ---------------------------------------------------------------------------------------------
struct ScoreSmem {
  ProbView v;
  OutWin win[TW_MAX_E];
  int64_t st_s[kStageSpans];
  int64_t st_e[kStageSpans];
  double prm[TW_MAX_TERMS * TW_MIX_REC];     // mixture table, or up to three Gaussian batch tables
  double tbl[kTblCap];                        // term tables of the in-spans of the current round
  uint8_t sid[kTblCap];                       // slot ids (term | batch << 6), TW_SLOT_INVALID
  uint32_t used[kWideThreads][TW_MAX_E][kWideW];
  int lo_abs[kWideThreads][TW_MAX_E];
  int win_a[TW_MAX_E], win_n[TW_MAX_E];
  int staged;
  int overflow;
  int rc;
  double etab[64];
};

// one wide tile (index t of `tiles`) by the whole CTA
__device__ __forceinline__ void score_tile(const tw_batch& b, const tw_params& prm, int has_params,
                                           const tw_score_out& out, const TileList& tiles, int t,
                                           const int32_t* __restrict__ prev_idx, int* __restrict__ err_flag,
                                           ScoreSmem& sm) {
  constexpr int T = kWideThreads;
  const int tid = threadIdx.x;
  int i0, cnt, p;
  for (int x = tid; x < 64; x += T) sm.etab[x] = c_exp2_64[x];   // visible after the barrier below
  p = tiles.tile_prob[t];
  i0 = tiles.tile_start[t];

  if (tid == 0) {
    sm.rc = load_view(b, p, sm.v);
    sm.overflow = 0;
  }
  __syncthreads();
  if (sm.rc != TW_OK) {
    if (tid == 0) atomicMin(err_flag, sm.rc);
    return;
  }
  const ProbView& v = sm.v;
  const int n = v.n_in;
  cnt = min(tiles.tile_cnt ? tiles.tile_cnt[t] : tiles.tile_len, n - i0);
  const int E = v.E;
  const bool helper = (tid == T - 1) && (i0 >= 1);
  const bool worker = tid < cnt;
  int i = i0 + tid;
  if (helper) i = prev_idx[v.in_off + i0];
  int64_t in_s = 0, in_e = INT64_MIN;
  if (worker || helper) { in_s = v.is[i]; in_e = v.ie[i]; }

  // ---- tile's candidate slice per ep: [lower_bound(start >= first in.start), upper_bound(start <= max in.end))
  int64_t me = worker ? in_e : INT64_MIN;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    int64_t o = __shfl_xor_sync(0xffffffffu, me, d);
    me = o > me ? o : me;
  }
  if (tid < E) {
    int a = lower_bound(v.os[tid], v.n_out[tid], v.is[i0]);
    int z = upper_bound(v.os[tid], v.n_out[tid], me);
    sm.win_a[tid] = a;
    sm.win_n[tid] = z > a ? z - a : 0;
  }
  __syncthreads();
  if (tid == 0) {
    int tot = 0;
    for (int e = 0; e < E; ++e) tot += sm.win_n[e];
    sm.staged = tot <= kStageSpans;
    int off = 0;
    for (int e = 0; e < E; ++e) {
      if (sm.staged) {
        sm.win[e].s = sm.st_s + off; sm.win[e].e = sm.st_e + off;
        sm.win[e].base = sm.win_a[e]; sm.win[e].n = sm.win_n[e];
        off += sm.win_n[e];
      } else {   // slice too large for shared memory: read the global arrays directly
        sm.win[e].s = v.os[e]; sm.win[e].e = v.oe[e]; sm.win[e].base = 0; sm.win[e].n = v.n_out[e];
      }
    }
  }
  __syncthreads();
  if (sm.staged) {
    for (int e = 0; e < E; ++e) {
      const int64_t* gs = v.os[e] + sm.win_a[e];
      const int64_t* ge = v.oe[e] + sm.win_a[e];
      int64_t* ds = const_cast<int64_t*>(sm.win[e].s);
      int64_t* de = const_cast<int64_t*>(sm.win[e].e);
      for (int x = tid; x < sm.win_n[e]; x += T) { ds[x] = gs[x]; de[x] = ge[x]; }
    }
  }
  // ---- likelihood parameters of this tile
  int batch0 = i0 / TW_PARAM_BATCH;
  if (has_params) {
    if (prm.mode == TW_PARAMS_GAUSS_BATCHED) {
      // a tile can touch three 100-span batches
      int nrec = 3 * v.n_terms * TW_GAUSS_REC;
      int nb = (n + TW_PARAM_BATCH - 1) / TW_PARAM_BATCH;
      const double* src = prm.gauss + (prm.prob_gauss_off[p] + (int64_t)batch0 * v.n_terms) * TW_GAUSS_REC;
      int avail = (nb - batch0) * v.n_terms * TW_GAUSS_REC;
      if (nrec > avail) nrec = avail;
      for (int x = tid; x < nrec; x += T) sm.prm[x] = src[x];
    } else {
      const double* src = prm.mix + (int64_t)v.term0 * TW_MIX_REC;
      for (int x = tid; x < v.n_terms * TW_MIX_REC; x += T) sm.prm[x] = src[x];
    }
  }
  for (int e = 0; e < TW_MAX_E; ++e)
    for (int wq = 0; wq < kWideW; ++wq) sm.used[tid][e][wq] = 0u;
  __syncthreads();

  // ---- per-thread first candidates
  OutWin w[TW_MAX_E];
  int lo[TW_MAX_E];
  const bool do_score = has_params && worker;
  if (worker || helper) {
    for (int e = 0; e < E; ++e) {
      if (helper && sm.staged) {   // carry-in span lies before the staged slice: use global arrays
        w[e].s = v.os[e]; w[e].e = v.oe[e]; w[e].base = 0; w[e].n = v.n_out[e];
      } else {
        w[e] = sm.win[e];
      }
      lo[e] = lower_bound(w[e].s, w[e].n, in_s);
      sm.lo_abs[tid][e] = w[e].base + lo[e];
    }
  }
  // candidate maps: a bit per candidate of the in-span (lane `owner`) from its first candidate on
  auto mark = [&](int owner, const int* c, const int* lo_abs, bool coop) {
    for (int e = 0; e < E; ++e) {
      const int bit = c[e] - lo_abs[e];
      if (bit >= 32 * kWideW) sm.overflow = 1;
      else if (coop) atomicOr(&sm.used[owner][e][bit >> 5], 1u << (bit & 31));
      else sm.used[owner][e][bit >> 5] |= 1u << (bit & 31);
    }
  };
  auto write_out = [&](const TopK& tk, int leaves) {
    int64_t gi = v.in_off + i;
    out.n_feasible[gi] = leaves;
    if (do_score && out.topk_score)
      store_topk_row(tk, E, out.topk_score + gi * TW_K, out.topk_idx + TW_K * (v.tuple_off + (int64_t)i * E),
                     out.topk_cnt + gi);
  };
  // windows-only launches and the carry-in helper only mark (no likelihoods)
  if ((worker || helper) && !do_score) {
    int leaves = 0;
    enumerate(v, in_s, in_e, w, lo, [](int, int) { return false; },
              [&](const int* c, const int64_t*, const int64_t*) {
                if (leaves < 0x7fffffff) ++leaves;
                mark(tid, c, sm.lo_abs[tid], false);
              });
    if (worker) { TopK none; none.clear(); write_out(none, leaves); }
  }
  // ---- scoring; every scored in-span is a worker, whose windows are the tile's staged ones
  auto params = [&](int bq) {   // the staged tables: mixtures, or the Gaussians of batch batch0 + bq
    return param_view(prm.mode, sm.prm, sm.prm, bq, v.n_terms, sm.etab);
  };
  warp_topk_search<kTblCap, kRedoCoopCombos>(v, sm.win, params, batch0, sm.tbl, sm.sid, tid, i, in_s, in_e, lo, do_score,
                                             [](int, int) { return false; }, mark, write_out);
  __syncthreads();

  // ---- PerfectCut(i), V3:1034-1039
  if (worker) {
    uint8_t cut = 0;
    if (i >= 1 && i <= n - 2) {
      int pi = prev_idx[v.in_off + i];
      int slot = pi >= i0 ? pi - i0 : T - 1;
      bool disjoint = true;
      for (int e = 0; e < E && disjoint; ++e)
        if (bitmaps_intersect(sm.used[slot][e], sm.lo_abs[slot][e], sm.used[tid][e], sm.lo_abs[tid][e], kWideW))
          disjoint = false;
      cut = (uint8_t)(disjoint && v.ie[pi] <= in_e);
    }
    out.cut[v.in_off + i] = cut;
    if (out.used_lo) out.used_wide[v.in_off + i] = 1;   // tw_stitch searches in-spans without narrow maps
  }
  if (tid == 0 && sm.overflow) atomicMin(err_flag, (int)TW_ERR_RANGE_LIMIT);
}

// A FIXED grid whose CTAs stride over the wide tiles and only work on those whose scoring tile was
// flagged (tiles.tile_start[n_tiles + t] = scoring tile of wide tile t): flagged tiles are rare, and
// one CTA per wide tile meant a quarter of a million CTAs that exit at once (1.9 ms per pass at 8192
// services).  The flags of 32 wide tiles are read at once (one coalesced load + one ballot), so a CTA
// mostly skims.
__global__ void __launch_bounds__(kWideThreads)
k_score(tw_batch b, tw_params prm, int has_params, tw_score_out out, TileList tiles,
        const int32_t* __restrict__ prev_idx, const uint8_t* __restrict__ overflow_flag, int* __restrict__ err_flag) {
  static_assert(kWideThreads == 32, "the redo kernel is written for one warp per CTA");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ScoreSmem& sm = *reinterpret_cast<ScoreSmem*>(smem_raw);
  for (int base = blockIdx.x * 32; base < tiles.n_tiles; base += gridDim.x * 32) {
    const int t0 = base + (int)threadIdx.x;
    const bool f = t0 < tiles.n_tiles && overflow_flag[tiles.tile_start[tiles.n_tiles + t0]] != 0;
    unsigned m = __ballot_sync(0xffffffffu, f);
    while (m) {
      const int t = base + __ffs(m) - 1;
      m &= m - 1u;
      score_tile(b, prm, has_params, out, tiles, t, prev_idx, err_flag, sm);
      __syncthreads();                                                    // shared memory is re-used
    }
  }
}

cudaError_t setup_score() {
  return cudaFuncSetAttribute(k_score, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ScoreSmem));
}

cudaError_t launch_score_redo(const tw_batch& b, const tw_params* prm, const tw_score_out& out,
                              const TileList& wide, const int32_t* prev_idx, uint8_t* tile_overflow,
                              int n_sm, int* err_flag, cudaStream_t s, int64_t& launches) {
  tw_params dummy;
  dummy.mode = TW_PARAMS_MIXTURE; dummy.reserved0 = 0;
  dummy.prob_gauss_off = nullptr; dummy.gauss = nullptr; dummy.mix = nullptr;
  const tw_params& pr = prm ? *prm : dummy;
  if (wide.n_tiles == 0) return cudaSuccess;
  const int chunks = (wide.n_tiles + 31) / 32;
  const int max_grid = 16 * n_sm;   // 16 CTAs per SM
  const int wide_grid = chunks < max_grid ? chunks : max_grid;
  k_score<<<wide_grid, kWideThreads, sizeof(ScoreSmem), s>>>(b, pr, prm != nullptr, out, wide, prev_idx,
                                                             tile_overflow, err_flag);
  return after_launch(launches);
}

}  // namespace tw
