// tw_score.cu — the SEQUENTIAL form of the scoring pass (one in-span per thread, depth-first
// enumeration, the reference's own tie order), used to redo the tiles the work-balanced kernel
// (tw_score3.cu) flags, plus the prev-index scan.  Candidate enumeration + likelihood scoring +
// top-K on the undeleted lists, and the perfect-cut flags.
//
// Replaces (reference: .../algorithms/traceweaver_v3.py = V3, traceweaver_v1.py = V1)
//   FindTopKAssignments(K=5, out_span_partitions)   V3:1185  (DfsTraverseX V3:292-351,
//       ScoreAssignmentAsPerInvocationGraph V1:259-361, GetEpPairCost V1:117-139)
//   CreateWindows2 pre-processing + PerfectCut       V3:1020-1051
//
// Mapping to the machine: HBM-bound integer/f64 work, no tensor cores.  One CTA owns a TILE of
// kScoreTile consecutive in-spans of one service (in-spans are sorted by start), one thread per
// in-span.  Because both sides are sorted by start, all candidates of the tile lie in one
// contiguous slice of each ep's out list: the slice's start/end timestamps are staged ONCE into
// shared memory (coalesced 128-bit loads) and every search / DFS step then runs out of shared
// memory; each out span is read from HBM about once per tile that overlaps it.  Likelihood
// parameters of the tile's one or two 100-span batches are staged alongside.  Thread
// kScoreThreads-1 enumerates the tile's carry-in "prev" in-span (the latest-ending in-span before
// the tile) so that PerfectCut(i) = disjoint(cand(prev(i)), cand(i)) is resolved inside the CTA
// from bitmaps in shared memory.  Tiles whose candidate ranges exceed the narrow bitmap width are
// flagged and redone by a wide instantiation (fewer threads, 2048 candidates per ep).
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
// score kernel
// ---------------------------------------------------------------------------------------------
template <int T, int W>
struct ScoreSmem {
  ProbView v;
  OutWin win[TW_MAX_E];
  int64_t st_s[kStageSpans];
  int64_t st_e[kStageSpans];
  double prm[TW_MAX_TERMS * TW_MIX_REC];     // mixture table, or up to three Gaussian batch tables
  double tbl[kTblCap];                        // term tables of the in-spans of the current round
  uint8_t sid[kTblCap];                       // slot ids (term | batch << 6), TW_SLOT_INVALID
  int scan[T / 32];
  int tbl_total;
  uint32_t used[T][TW_MAX_E][W];
  int lo_abs[T][TW_MAX_E];
  int64_t red[T / 32];
  int win_a[TW_MAX_E], win_n[TW_MAX_E];
  int staged;
  int overflow;
  int rc;
  double etab[64];
};

// one tile (index t of `tiles`) by the whole CTA
template <int T, int W>
__device__ __forceinline__ void score_tile(const tw_batch& b, const tw_params& prm, int has_params,
                                           const tw_score_out& out, const TileList& tiles, int t,
                                           const int32_t* __restrict__ prev_idx,
                                           uint8_t* __restrict__ overflow_flag, int redo_only,
                                           int* __restrict__ err_flag, ScoreSmem<T, W>& sm) {
  const int tid = threadIdx.x;
  int i0, cnt, p;
  for (int x = tid; x < 64; x += T) sm.etab[x] = c_exp2_64[x];   // (T may be 32) visible after the barrier below
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
  if ((tid & 31) == 0) sm.red[tid >> 5] = me;
  __syncthreads();
  if (tid < E) {
    int64_t mx = sm.red[0];
    for (int q = 1; q < T / 32; ++q) mx = sm.red[q] > mx ? sm.red[q] : mx;
    int a = lower_bound(v.os[tid], v.n_out[tid], v.is[i0]);
    int z = upper_bound(v.os[tid], v.n_out[tid], mx);
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
    for (int wq = 0; wq < W; ++wq) sm.used[tid][e][wq] = 0u;
  __syncthreads();

  // ---- per-thread candidate ranges
  OutWin w[TW_MAX_E];
  int lo[TW_MAX_E], r[TW_MAX_E];
  int tsize = 0;
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
      r[e] = do_score ? range_len(w[e], lo[e], in_e) : 0;
    }
    if (do_score) tsize = term_table_size(v, r);
  }
  uint32_t (*mine)[W] = sm.used[tid];
  const int* lo_abs = sm.lo_abs[tid];
  auto mark = [&](const int* c, bool& ovf) {
    for (int e = 0; e < E; ++e) {
      int bit = c[e] - lo_abs[e];
      if (bit >= 32 * W) ovf = true;
      else mine[e][bit >> 5] |= 1u << (bit & 31);
    }
  };
  auto write_out = [&](const TopK& tk, int leaves) {
    int64_t gi = v.in_off + i;
    out.n_feasible[gi] = leaves;
    if (do_score && out.topk_score) {
      out.topk_cnt[gi] = (uint8_t)tk.n;
      int32_t* ix = out.topk_idx + TW_K * (v.tuple_off + (int64_t)i * E);
      for (int k = 0; k < TW_K; ++k) {
        out.topk_score[gi * TW_K + k] = k < tk.n ? tk.score[k] : __longlong_as_double(0x7ff8000000000000LL);
        for (int e = 0; e < E; ++e) ix[k * E + e] = k < tk.n ? tk.idx[k][e] : -1;
      }
    }
  };
  // windows-only launches and the carry-in helper only mark (no likelihoods)
  if ((worker || helper) && !do_score) {
    int leaves = 0;
    bool ovf = false;
    enumerate(v, in_s, in_e, w, lo, [](int, int) { return false; },
              [&](const int* c, const int64_t*, const int64_t*) {
                if (leaves < 0x7fffffff) ++leaves;
                mark(c, ovf);
              });
    if (ovf) sm.overflow = 1;
    if (worker) { TopK none; none.clear(); write_out(none, leaves); }
  }
  // ---- scoring: term tables in shared memory, evaluated by the whole CTA (see tw_core.cuh)
  if (has_params) {
    bool pending = do_score;
    const int lane = tid & 31, wid = tid >> 5;
    // ---- heavy in-spans, one at a time by the WHOLE warp (one-warp CTAs only: the redo kernel).  A thread
    // that walks thousands of tuples alone keeps one lane of 32 busy and sets the kernel's time; here the
    // owner lays out its term tables, all lanes evaluate the slots, then take the combinations lane,
    // lane + 32, ... (ascending combination index = depth-first leaf order), mark the candidate maps, keep
    // their own top K, and the warp merges the heads.  Two equal scores among the best -> the reference's
    // heap order decides (topk_offer): the in-span stays pending and its owner redoes it alone below.
    if (T == 32) {
      const long long Pown = pending ? combo_count(v, r) : 0;
      unsigned heavy = __ballot_sync(0xffffffffu, pending && tsize <= kTblCap && Pown > kRedoCoopCombos &&
                                                      Pown < (1LL << 31));
      const int brel_own = i / TW_PARAM_BATCH - batch0;
      while (heavy) {
        const int L = __ffs(heavy) - 1;
        heavy &= heavy - 1u;
        int lo_b[TW_MAX_E], r_b[TW_MAX_E], o_last_b[TW_MAX_E], lo_abs_b[TW_MAX_E];
        for (int e = 0; e < E; ++e) {
          lo_b[e] = __shfl_sync(0xffffffffu, lo[e], L);
          r_b[e] = __shfl_sync(0xffffffffu, r[e], L);
          lo_abs_b[e] = sm.lo_abs[L][e];
        }
        const int tsz = __shfl_sync(0xffffffffu, tsize, L);
        const long long P_b = __shfl_sync(0xffffffffu, Pown, L);
        term_table_last_offsets(v, r_b, o_last_b);
        if (lane == L)
          term_table_fill(v, in_s, in_e, w, lo, r, o_last_b, brel_own, [](int, int) { return false; }, sm.tbl, sm.sid);
        __syncwarp();
        for (int sl = lane; sl < tsz; sl += 32) {
          const uint8_t id = sm.sid[sl];
          if (id != TW_SLOT_INVALID) {
            ParamView pv;
            pv.mode = prm.mode;
            pv.gauss = sm.prm + (id >> 6) * v.n_terms * TW_GAUSS_REC;
            pv.mix = sm.prm;
            pv.etab = sm.etab;
            sm.tbl[sl] = term_logpdf(pv, id & 63, sm.tbl[sl]);
          }
        }
        __syncwarp();
        TopK part;
        part.clear();
        int leaves = 0;
        bool tie = false, ovf = false;
        enumerate_combos(v, sm.win, lo_b, r_b, o_last_b, sm.sid, lane, 32, P_b,
                         [&](const int* c, const int64_t* ce, long long) {
                           ++leaves;
                           for (int e = 0; e < E; ++e) {
                             const int bit = c[e] - lo_abs_b[e];
                             if (bit >= 32 * W) ovf = true;
                             else atomicOr(&sm.used[L][e][bit >> 5], 1u << (bit & 31));
                           }
                           const double sc = table_score(v, r_b, lo_abs_b, sm.tbl, c, ce);
                           for (int k = 0; k < part.n; ++k) tie = tie || part.score[k] == sc;
                           tie = tie || sc != sc;
                           topk_offer_sorted(v, part, sc, c);
                         });
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) leaves += __shfl_xor_sync(0xffffffffu, leaves, d);
        if (ovf) sm.overflow = 1;
        TopK tkc;
        tkc.clear();
        int head = 0;
        double prev = 0.0;
        for (int round = 0; round <= TW_K; ++round) {
          const double hs = head < part.n ? part.score[head] : -INFINITY;
          double mx = hs;
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) {
            const double o = __shfl_xor_sync(0xffffffffu, mx, d);
            mx = o > mx ? o : mx;
          }
          if (!(mx > -INFINITY)) break;
          const unsigned who = __ballot_sync(0xffffffffu, hs == mx);
          if (__popc(who) > 1 || (round > 0 && mx == prev)) tie = true;
          prev = mx;
          const int wl = __ffs(who) - 1;
          if (round < TW_K) {
            for (int e = 0; e < E; ++e) {
              const int ci = __shfl_sync(0xffffffffu, head < part.n ? part.idx[head][e] : -1, wl);
              if (lane == L) tkc.idx[round][e] = ci;
            }
            if (lane == L) { tkc.score[round] = mx; tkc.n = round + 1; }
          }
          if (lane == wl) ++head;
        }
        tie = __any_sync(0xffffffffu, tie);
        if (!tie && lane == L) {
          write_out(tkc, leaves);
          pending = false;
        }
        __syncwarp();
      }
    }
    while (true) {
      // exclusive prefix of the pending threads' table sizes
      int my = pending ? tsize : 0, incl = my;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
      }
      if (lane == 31) sm.scan[wid] = incl;
      if (tid == 0) sm.tbl_total = 0;
      __syncthreads();
      int offset = incl - my;
      for (int q = 0; q < wid; ++q) offset += sm.scan[q];
      const bool lazy = pending && offset == 0 && tsize > kTblCap;     // does not fit at all
      const bool in_round = pending && !lazy && offset + tsize <= kTblCap;
      int o_last[TW_MAX_E];
      const int brel = i / TW_PARAM_BATCH - batch0;
      if (in_round) {
        term_table_last_offsets(v, r, o_last);
        term_table_fill(v, in_s, in_e, w, lo, r, o_last, brel, [](int, int) { return false; }, sm.tbl + offset,
                        sm.sid + offset);
        atomicMax(&sm.tbl_total, offset + tsize);
      }
      if (lazy) {   // per-leaf evaluation for an in-span whose tables exceed shared memory
        ParamView pv;
        pv.mode = prm.mode;
        pv.gauss = sm.prm + brel * v.n_terms * TW_GAUSS_REC;
        pv.mix = sm.prm;
        pv.etab = sm.etab;
        TopK tk;
        tk.clear();
        int leaves = 0;
        bool ovf = false;
        enumerate(v, in_s, in_e, w, lo, [](int, int) { return false; },
                  [&](const int* c, const int64_t* cs, const int64_t* ce) {
                    if (leaves < 0x7fffffff) ++leaves;
                    mark(c, ovf);
                    topk_offer(v, tk, score_tuple(v, pv, in_s, in_e, cs, ce), c);
                  });
        if (ovf) sm.overflow = 1;
        topk_finish(v, tk);
        write_out(tk, leaves);
        pending = false;
      }
      __syncthreads();
      // dense pass: every lane evaluates slots (GetEpPairCost, V1:117-139)
      const int total = sm.tbl_total;
      for (int s = tid; s < total; s += T) {
        const uint8_t id = sm.sid[s];
        if (id != TW_SLOT_INVALID) {
          ParamView pv;
          pv.mode = prm.mode;
          pv.gauss = sm.prm + (id >> 6) * v.n_terms * TW_GAUSS_REC;
          pv.mix = sm.prm;
          pv.etab = sm.etab;
          sm.tbl[s] = term_logpdf(pv, id & 63, sm.tbl[s]);
        }
      }
      __syncthreads();
      if (in_round) {
        const double* tbl = sm.tbl + offset;
        const uint8_t* sid = sm.sid + offset;
        TopK tk;
        tk.clear();
        int leaves = 0;
        bool ovf = false;
        enumerate(v, in_s, in_e, w, lo,
                  [&](int e, int o) { return sid[o_last[e] + (o - lo_abs[e])] == TW_SLOT_INVALID; },
                  [&](const int* c, const int64_t*, const int64_t* ce) {
                    if (leaves < 0x7fffffff) ++leaves;
                    mark(c, ovf);
                    topk_offer(v, tk, table_score(v, r, lo_abs, tbl, c, ce), c);
                  });
        if (ovf) sm.overflow = 1;
        topk_finish(v, tk);
        write_out(tk, leaves);
        pending = false;
      }
      if (!__syncthreads_or(pending)) break;
    }
  }
  __syncthreads();

  // ---- PerfectCut(i), V3:1034-1039
  if (worker) {
    uint8_t cut = 0;
    if (i >= 1 && i <= n - 2) {
      int pi = prev_idx[v.in_off + i];
      int slot = pi >= i0 ? pi - i0 : T - 1;
      bool disjoint = true;
      for (int e = 0; e < E && disjoint; ++e)
        if (bitmaps_intersect(sm.used[slot][e], sm.lo_abs[slot][e], sm.used[tid][e], sm.lo_abs[tid][e], W))
          disjoint = false;
      cut = (uint8_t)(disjoint && v.ie[pi] <= in_e);
    }
    out.cut[v.in_off + i] = cut;
    if (out.used_lo) {   // candidate maps for tw_stitch's "nothing taken" proof
      const int64_t base = v.tuple_off + (int64_t)i * E;
      if (W == kNarrowW) {
        for (int e = 0; e < E; ++e) {
          out.used_lo[base + e] = sm.lo_abs[tid][e];
          out.used_bits[2 * (base + e)] = sm.used[tid][e][0];
          out.used_bits[2 * (base + e) + 1] = sm.used[tid][e][1];
        }
        out.used_wide[v.in_off + i] = 0;
      } else {
        out.used_wide[v.in_off + i] = 1;
      }
    }
  }
  if (tid == 0 && sm.overflow) {
    if (redo_only) atomicMin(err_flag, (int)TW_ERR_RANGE_LIMIT);
    else overflow_flag[t] = 1;
  }
}

// Normal launches: CTA t owns tile t.  The wide redo pass (redo_only) runs a FIXED grid whose CTAs
// stride over the wide tiles and only work on those whose narrow tile overflowed
// (tiles.tile_start[n_tiles + t] = narrow tile of wide tile t): overflow is rare, and one CTA per
// wide tile meant a quarter of a million CTAs that exit at once (1.9 ms per pass at 8192 services).
template <int T, int W>
__global__ void __launch_bounds__(T)
k_score(tw_batch b, tw_params prm, int has_params, tw_score_out out, TileList tiles,
        const int32_t* __restrict__ prev_idx, uint8_t* __restrict__ overflow_flag, int redo_only,
        int* __restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ScoreSmem<T, W>& sm = *reinterpret_cast<ScoreSmem<T, W>*>(smem_raw);
  if (!redo_only) {
    score_tile<T, W>(b, prm, has_params, out, tiles, blockIdx.x, prev_idx, overflow_flag, 0, err_flag, sm);
    return;
  }
  // the flags of T wide tiles are read at once (one coalesced load + one ballot per 32); flagged
  // tiles are rare, so a CTA mostly skims
  static_assert(T == 32, "the redo scan is written for one warp per CTA");
  for (int base = blockIdx.x * 32; base < tiles.n_tiles; base += gridDim.x * 32) {
    const int t0 = base + (int)threadIdx.x;
    const bool f = t0 < tiles.n_tiles && overflow_flag[tiles.tile_start[tiles.n_tiles + t0]] != 0;
    unsigned m = __ballot_sync(0xffffffffu, f);
    while (m) {
      const int t = base + __ffs(m) - 1;
      m &= m - 1u;
      score_tile<T, W>(b, prm, has_params, out, tiles, t, prev_idx, overflow_flag, 1, err_flag, sm);
      __syncthreads();                                                    // shared memory is re-used
    }
  }
}

using SmW = ScoreSmem<kWideThreads, kWideW>;

cudaError_t setup_score() {
  return cudaFuncSetAttribute(k_score<kWideThreads, kWideW>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)sizeof(SmW));
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
  k_score<kWideThreads, kWideW><<<wide_grid, kWideThreads, sizeof(SmW), s>>>(b, pr, prm != nullptr, out, wide,
                                                                            prev_idx, tile_overflow, 1, err_flag);
  return after_launch(launches);
}

}  // namespace tw
