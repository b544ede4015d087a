// tw_stitch.cu — the sequential half of one pass: windows, per in-span top-K on the not-yet-taken
// out spans, exact MWIS per window, assignment + deletion.
//
// Replaces (V3 = traceweaver_v3.py, V1 = traceweaver_v1.py)
//   window loop                      V3:1056-1076 (from the cut flags of tw_score.cu)
//   FindTopKAssignments(out_copy)    V3:1182
//   GetAssignmentsMIS / Gurobi_MIS   V3:1237-1274, 1395-1419
//   AddAssignment(delete=True)       V1:433-463   -> "taken" bitmap instead of list.remove
//
// Window w's candidates exclude out spans consumed by windows < w, so a service is a sequential
// chain of windows; services are independent.  One WARP owns one service and walks its windows in
// order: lane l enumerates + scores in-span (window start + l) (a window holds <= 31 in-spans),
// the candidates meet in shared memory, lanes build the in-span conflict masks in parallel, lane 0
// runs the exact branch and bound, lanes write assignments and set taken bits.  Parallelism comes
// from the number of services in the batch (25 000 in the 100 M-span configuration).
#include "tw_kernels.cuh"

namespace tw {

// optional phase timers (build with -DTW_PROFILE_PHASES; scripts/stitch_phase_profile.py reads them)
#ifdef TW_PROFILE_PHASES
__device__ unsigned long long g_stitch_phase[16];
#define TW_SPHASE(k)                                                                 \
  do {                                                                               \
    if (lane == 0) {                                                                 \
      long long _now = clock64();                                                    \
      atomicAdd(&g_stitch_phase[k], (unsigned long long)(_now - _sp_t0));            \
      _sp_t0 = _now;                                                                 \
    }                                                                                \
  } while (0)
#define TW_SCOUNT(k, v) do { if (lane == 0) atomicAdd(&g_stitch_phase[k], (unsigned long long)(v)); } while (0)
#else
#define TW_SPHASE(k) do { } while (0)
#define TW_SCOUNT(k, v) do { } while (0)
#endif

__device__ __forceinline__ void prefetch_l1(const void* p) {
  asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
}

// Fixed part of a warp's slab; the rest is laid out per batch (StitchLayout, stitch_layout):
//   uint32_t tk[tk_words]     taken bitmap of the service when it fits (else global memory)
//   uint32_t tmp[tk_words]    scratch bitmap of the run path (always left zero)
//   PackedWindowBuf           at wb_off, the tuple planes of the batch's largest E
struct StitchWarpSmem {
  ProbView v;
  uint32_t cconf[32];          // small-window solver: conflict mask / weight of candidate lane 5k + r
  double cw[32];
};
static_assert(sizeof(StitchWarpSmem) % 8 == 0, "the taken bitmaps and the window buffer follow 8-byte aligned");

// The slab of one warp and the pointers into it; every access to the per-batch part goes through here.
struct StitchSlab {
  unsigned char* base;
  __device__ StitchWarpSmem& fixed() const { return *reinterpret_cast<StitchWarpSmem*>(base); }
  __device__ uint32_t* taken() const { return reinterpret_cast<uint32_t*>(base + sizeof(StitchWarpSmem)); }
  __device__ PackedWindowBuf& window(const StitchLayout& L) const {
    return *reinterpret_cast<PackedWindowBuf*>(base + L.wb_off);
  }
};

// Exact MWIS of a window of <= kSmallWindow in-spans by the whole warp (the search and its tie rule:
// tw_core.cuh, small_component .. SmallBest).  Here is what the warp does together: the conflicts of
// candidate lane 5k + r with the other candidates come from one __match_any_sync per tuple position
// (AssignmentIntersect, V3:1276-1281), the lanes take the leaves lane, lane + 32, ... of a component
// and an xor butterfly merges their bests.  Returns false (nothing decided) when a component needs
// the sequential solver: E == 1 with >= 3 in-spans (Hungarian path) or more than kSmallSpace leaves.
__device__ __forceinline__ bool stitch_small_window(StitchWarpSmem& sm, PackedWindowBuf& wb, int E, int nw, int lane,
                                                    long long* nodes_out) {
  const unsigned kAll = 0xffffffffu;
  const int k = lane / TW_K, r = lane - TW_K * k;
  const bool valid = k < nw && r < wb.cnt[k];
  const unsigned vmask = __ballot_sync(kAll, valid);
  uint32_t conf = 0u;
  if (valid) {
    for (int e = 0; e < E; ++e) conf |= __match_any_sync(vmask, wb.at(k, r, e));
    conf &= ~(0x1fu << (TW_K * k));
  }
  sm.cconf[lane] = conf;
  sm.cw[lane] = valid ? TW_WEIGHT_OFFSET + wb.score[k][r] : 0.0;
  uint32_t am = 0u;
#pragma unroll
  for (int a = 0; a < kSmallWindow; ++a)
    if ((conf >> (TW_K * a)) & 0x1fu) am |= 1u << a;
  if (lane < nw) { wb.adj[lane] = 0u; wb.chosen[lane] = -1; }
  __syncwarp();
  if (am) atomicOr(&wb.adj[k], am);
  __syncwarp();
  int cnt[kSmallWindow];
  uint32_t adj[kSmallWindow];
#pragma unroll
  for (int a = 0; a < kSmallWindow; ++a) { cnt[a] = a < nw ? wb.cnt[a] : 0; adj[a] = a < nw ? wb.adj[a] : 0u; }
  long long nodes = 0;
  uint32_t todo = (1u << nw) - 1u;
  while (todo) {
    const int seed = lowest_bit(todo);
    const uint32_t comp = small_component(adj, seed);
    todo &= ~comp;
    const int m = __popc(comp);
    if (m == 1) {   // isolated in-span: its best candidate, if the weight is positive
      if (lane == 0 && wb.cnt[seed] > 0 && sm.cw[TW_K * seed] > 0.0) wb.chosen[seed] = 0;
      ++nodes;
      continue;
    }
    if (E == 1 && m >= 3) return false;
    int stride[kSmallWindow];
    const int space = small_strides(comp, cnt, stride);
    if (space > kSmallSpace) return false;
    SmallBest best;
    for (int idx = lane; idx < space; idx += 32) {
      double tot;
      if (small_leaf(comp, cnt, stride, sm.cw, sm.cconf, idx, &tot)) best.offer(tot, idx);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      SmallBest other;
      other.w = __shfl_xor_sync(kAll, best.w, d);
      other.idx = __shfl_xor_sync(kAll, best.idx, d);
      best.merge(other);
    }
    small_decode(comp, cnt, stride, best.idx, [&](int a, int rank) {
      if (lane == 0) wb.chosen[a] = rank;
    });
    nodes += space;
  }
  *nodes_out = nodes;
  return true;
}


// Priced branch and bound of ONE connected component by the whole warp (the sequential form is
// mwis_solve's second search, tw_core.cuh: same order, same bounds, same tie rule).  Lane l owns the
// l-th in-span of the component: its availability mask per level, its weights and prices.  A node is
// expanded by all lanes at once — the owner's choice is broadcast, every later in-span strikes its
// conflicting ranks, two warp sums give the bounds of the child — so a node costs tens of
// instructions instead of the hundreds of the one-lane loop over (in-span, rank, tuple position).
// `price` (the warp's StitchTables): dual prices of one callee's assignment relaxation, written by lane 0.
__device__ __noinline__ long long mwis_component_warp(PackedWindowBuf& wb, int E, uint32_t comp, double* price /*[31][TW_K]*/,
                                                      long long node_limit, long long nodes, int lane) {
  const unsigned kAll = 0xffffffffu;
  // members in window order
  const int m = __popc(comp);
  int kmine = -1;                                   // own in-span (window index)
  {
    uint32_t c = comp;
    for (int l = 0; l < m; ++l) {
      const int k = __ffs(c) - 1;
      c &= c - 1u;
      if (l == lane) kmine = k;
    }
  }
  // ---- prices: lane 0 solves the relaxation (callee with the fewest distinct spans)
  double lam0 = 0.0;
  if (lane == 0) {
    int member[TW_WINDOW_CAP];
    {
      uint32_t c = comp;
      for (int l = 0; l < m; ++l) { member[l] = __ffs(c) - 1; c &= c - 1u; }
    }
    int pos = 0, fewest = 0x7fffffff;
    for (int e = 0; e < E; ++e) {
      int distinct = 0;
      for (int l = 0; l < m; ++l)
        for (int r = 0; r < wb.cnt[member[l]]; ++r) {
          const int sp = wb.at(member[l], r, e);
          bool seen = false;
          for (int l2 = 0; l2 <= l && !seen; ++l2)
            for (int r2 = 0; r2 < (l2 < l ? wb.cnt[member[l2]] : r) && !seen; ++r2)
              seen = wb.at(member[l2], r2, e) == sp;
          distinct += !seen;
        }
      if (distinct < fewest) { fewest = distinct; pos = e; }
    }
    assignment_solve(wb, member, m, pos, nullptr, reinterpret_cast<double(*)[TW_K]>(price), &lam0);
  }
  __syncwarp();
  lam0 = __shfl_sync(kAll, lam0, 0);
  nodes += m;
  const bool mine = lane < m;
  const int cnt = mine ? wb.cnt[kmine] : 0;
  double w0 = 0, w1 = 0, w2 = 0, w3 = 0, w4 = 0, q0 = 0, q1 = 0, q2 = 0, q3 = 0, q4 = 0;   // weights, reduced weights
  uint8_t av[TW_WINDOW_CAP + 1];
  {
    uint8_t mask = 0;
    if (mine) {
      double wv[TW_K], qv[TW_K];
      for (int r = 0; r < TW_K; ++r) {
        wv[r] = r < cnt ? TW_WEIGHT_OFFSET + wb.score[kmine][r] : 0.0;
        qv[r] = wv[r] - price[lane * TW_K + r];
        if (r < cnt && wv[r] > 0.0) mask |= (uint8_t)(1u << r);
      }
      w0 = wv[0]; w1 = wv[1]; w2 = wv[2]; w3 = wv[3]; w4 = wv[4];
      q0 = qv[0]; q1 = qv[1]; q2 = qv[2]; q3 = qv[3]; q4 = qv[4];
    }
    av[0] = mask;
  }
  auto best_avail = [&](uint8_t mask) {           // lists are sorted: the lowest available rank is the heaviest
    return (mask & 1u) ? w0 : (mask & 2u) ? w1 : (mask & 4u) ? w2 : (mask & 8u) ? w3 : (mask & 16u) ? w4 : 0.0;
  };
  auto best_reduced = [&](uint8_t mask) {
    double mx = 0.0;
    if ((mask & 1u) && q0 > mx) mx = q0;
    if ((mask & 2u) && q1 > mx) mx = q1;
    if ((mask & 4u) && q2 > mx) mx = q2;
    if ((mask & 8u) && q3 > mx) mx = q3;
    if ((mask & 16u) && q4 > mx) mx = q4;
    return mx;
  };
  auto wsum = [&](double x) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(kAll, x, d);
    return x;
  };
  double cur[TW_WINDOW_CAP + 1], rem[TW_WINDOW_CAP + 1], remp[TW_WINDOW_CAP + 1], lam[TW_WINDOW_CAP + 1];
  int8_t iter[TW_WINDOW_CAP + 1];
  rem[0] = wsum(best_avail(av[0]));
  remp[0] = wsum(best_reduced(av[0]));
  lam[0] = lam0;
  cur[0] = 0.0;
  iter[0] = 0;
  int myc = -1, bestc = -1;
  double best_w = -1.0;
  int level = 0;
  while (level >= 0) {
    if (level == m) {
      ++nodes;
      if (cur[m] > best_w + TW_MWIS_TIE_TOL) { best_w = cur[m]; bestc = myc; }   // a tied total never replaces an earlier leaf
      --level;
      continue;
    }
    if (iter[level] == 0) {
      ++nodes;
      if (node_limit > 0 && nodes > node_limit) return -1;
      double bound = rem[level] + 1e-7;
      const double bp = remp[level] + lam[level] + 1e-7;
      bound = bp < bound ? bp : bound;
      if (cur[level] + bound <= best_w + TW_MWIS_TIE_TOL) { --level; continue; }
    }
    const int r = iter[level]++;
    const int cntL = __shfl_sync(kAll, cnt, level);
    if (r > cntL) { --level; continue; }
    const uint8_t avmine = av[level];
    const unsigned avL = __shfl_sync(kAll, (unsigned)avmine, level);
    if (r == cntL) {                                // leave the in-span unassigned
      const double ob = __shfl_sync(kAll, best_avail(avmine), level);
      const double obp = __shfl_sync(kAll, best_reduced(avmine), level);
      if (lane == level) myc = -1;
      av[level + 1] = avmine;
      cur[level + 1] = cur[level];
      rem[level + 1] = rem[level] - ob;
      remp[level + 1] = remp[level] - obp;
      lam[level + 1] = lam[level];
      ++level;
      iter[level] = 0;
      continue;
    }
    if (!(avL >> r & 1u)) continue;                 // weight <= 0, or struck by an earlier choice
    const int kL = __shfl_sync(kAll, kmine, level);
    uint8_t mask = avmine;
    if (mine && lane > level && mask && (wb.adj[kL] >> kmine & 1u)) {
      for (int q = 0; q < cnt; ++q)
        if ((mask >> q & 1u) && cands_conflict(wb, kL, r, kmine, q, E)) mask &= (uint8_t)~(1u << q);
    }
    av[level + 1] = mask;
    const bool later = mine && lane > level;
    const double rest = wsum(later ? best_avail(mask) : 0.0);
    const double restp = wsum(later ? best_reduced(mask) : 0.0);
    if (lane == level) myc = r;
    cur[level + 1] = cur[level] + (TW_WEIGHT_OFFSET + wb.score[kL][r]);
    rem[level + 1] = rest;
    remp[level + 1] = restp;
    lam[level + 1] = lam[level] - price[level * TW_K + r];
    ++level;
    iter[level] = 0;
  }
  if (mine) wb.chosen[kmine] = bestc;
  __syncwarp();
  return nodes;
}

// Search path of one window: the lanes flagged `todo` enumerate + score their in-span on the
// not-yet-taken out spans (term tables in the warp's StitchTables, evaluated by all lanes) and leave
// their top-K lists in the window buffer.  Out of line on purpose: it is large and rarely taken (an
// in-span gets here only when one of its candidates was taken by an earlier window).
__device__ __noinline__ void stitch_search_lanes(const ProbView& v, PackedWindowBuf& wb, StitchTables& tb,
                                                 const tw_params& prm, const tw_pass_out& out,
                                                 uint32_t* const* tk_base, const OutWin* w,
                                                 const double* gauss_base, const double* mix_base, const double* etab,
                                                 int E, int lane, int ws, int i, int64_t in_s, int64_t in_e,
                                                 bool todo, int batch0) {
  auto is_taken = [&](int e, int o) {   // volatile: bits are set by other lanes with atomics
    return (reinterpret_cast<volatile const uint32_t*>(tk_base[e])[o >> 5] >> (o & 31)) & 1u;
  };
  const bool active = todo, fast = false;
  int lo[TW_MAX_E], r[TW_MAX_E], lo_abs[TW_MAX_E];
  int tsize = 0;
  if (active && !fast) {
    for (int e = 0; e < E; ++e) {
      lo[e] = lower_bound(w[e].s, w[e].n, in_s);
      lo_abs[e] = lo[e];
      r[e] = range_len(w[e], lo[e], in_e);
    }
    tsize = term_table_size(v, r);
  }
  const int brel = i / TW_PARAM_BATCH - batch0;
  auto publish = [&](const TopK& tk, int leaves) {
    const int64_t gi = v.in_off + i;
    out.n_cand[gi] = leaves;
    wb.cnt[lane] = tk.n;
    for (int k = 0; k < tk.n; ++k) {
      wb.score[lane][k] = tk.score[k];
      for (int e = 0; e < E; ++e) wb.at(lane, k, e) = tk.idx[k][e];
    }
    if (out.topk_score)
      store_topk_row(tk, E, out.topk_score + gi * TW_K, out.topk_idx + TW_K * (v.tuple_off + (int64_t)i * E),
                     out.topk_cnt + gi);
  };
  bool pending = active;
  // ---- heavy in-spans (thousands of candidate combinations), one at a time by the WHOLE warp:
  // the owner lays out its term tables, all lanes evaluate the slots, then the lanes take the
  // combinations lane, lane + 32, ... (ascending combination index = depth-first leaf order), keep
  // their own top K and the warp merges the heads.  If two of the six best scores are equal the
  // reference's heap order decides (tw_core.cuh topk_offer) and the owner redoes the in-span alone.
  {
    const long long Pown = pending ? combo_count(v, r) : 0;
    unsigned heavy = __ballot_sync(0xffffffffu, pending && tsize <= kWarpTblCap && Pown > kStitchCoopCombos &&
                                                    Pown < (1LL << 31));
    while (heavy) {
      const int L = __ffs(heavy) - 1;
      heavy &= heavy - 1u;
      int lo_b[TW_MAX_E], r_b[TW_MAX_E], o_last_b[TW_MAX_E];
      for (int e = 0; e < E; ++e) {
        lo_b[e] = __shfl_sync(0xffffffffu, lo[e], L);
        r_b[e] = __shfl_sync(0xffffffffu, r[e], L);
      }
      const int tsz = __shfl_sync(0xffffffffu, tsize, L);
      const int brel_b = __shfl_sync(0xffffffffu, brel, L);
      const long long P_b = __shfl_sync(0xffffffffu, Pown, L);
      term_table_last_offsets(v, r_b, o_last_b);
      if (lane == L) term_table_fill(v, in_s, in_e, w, lo, r, o_last_b, brel_b, is_taken, tb.tbl, tb.sid);
      __syncwarp();
      for (int sl = lane; sl < tsz; sl += 32) {
        const uint8_t id = tb.sid[sl];
        if (id != TW_SLOT_INVALID)
          tb.tbl[sl] = term_logpdf(param_view(prm.mode, gauss_base, mix_base, batch0 + (id >> 6), v.n_terms, etab),
                                   id & 63, tb.tbl[sl]);
      }
      __syncwarp();
      TopK part;
      part.clear();
      int leaves = 0;
      bool tie = false;
      enumerate_combos(v, w, lo_b, r_b, o_last_b, tb.sid, lane, 32, P_b,
                       [&](const int* c, const int64_t* ce, long long) {
                         ++leaves;
                         const double sc = table_score(v, r_b, lo_b, tb.tbl, c, ce);
                         for (int k = 0; k < part.n; ++k) tie = tie || part.score[k] == sc;
                         tie = tie || sc != sc;
                         topk_offer_sorted(v, part, sc, c);
                       });
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) leaves += __shfl_xor_sync(0xffffffffu, leaves, d);
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
        publish(tkc, leaves);
        pending = false;
      }
      __syncwarp();
    }
  }
  if (__any_sync(0xffffffffu, pending))
  while (true) {
    int my = pending ? tsize : 0, incl = my;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += o;
    }
    const int offset = incl - my;
    const bool lazy = pending && offset == 0 && tsize > kWarpTblCap;
    const bool in_round = pending && !lazy && offset + tsize <= kWarpTblCap;
    int total = in_round ? offset + tsize : 0;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) total = max(total, __shfl_xor_sync(0xffffffffu, total, d));
    int o_last[TW_MAX_E];
    if (in_round) {
      term_table_last_offsets(v, r, o_last);
      term_table_fill(v, in_s, in_e, w, lo, r, o_last, brel, is_taken, tb.tbl + offset, tb.sid + offset);
    }
    if (lazy) {   // tables larger than the warp's StitchTables: evaluate per leaf
      const ParamView pv = param_view(prm.mode, gauss_base, mix_base, i / TW_PARAM_BATCH, v.n_terms, etab);
      TopK tk;
      tk.clear();
      int leaves = 0;
      enumerate(v, in_s, in_e, w, lo, is_taken,
                [&](const int* c, const int64_t* cs, const int64_t* ce) {
                  if (leaves < 0x7fffffff) ++leaves;
                  topk_offer(v, tk, score_tuple(v, pv, in_s, in_e, cs, ce), c);
                });
      topk_finish(v, tk);
      publish(tk, leaves);
      pending = false;
    }
    __syncwarp();
    for (int s = lane; s < total; s += 32) {     // GetEpPairCost for every slot, all lanes busy
      const uint8_t id = tb.sid[s];
      if (id != TW_SLOT_INVALID)
        tb.tbl[s] = term_logpdf(param_view(prm.mode, gauss_base, mix_base, batch0 + (id >> 6), v.n_terms, etab),
                                id & 63, tb.tbl[s]);
    }
    __syncwarp();
    if (in_round) {
      const double* tbl = tb.tbl + offset;
      const uint8_t* sid = tb.sid + offset;
      TopK tk;
      tk.clear();
      int leaves = 0;
      enumerate(v, in_s, in_e, w, lo,
                [&](int e, int o) { return sid[o_last[e] + (o - lo_abs[e])] == TW_SLOT_INVALID; },
                [&](const int* c, const int64_t*, const int64_t* ce) {
                  if (leaves < 0x7fffffff) ++leaves;
                  topk_offer(v, tk, table_score(v, r, lo_abs, tbl, c, ce), c);
                });
      topk_finish(v, tk);
      publish(tk, leaves);
      pending = false;
    }
    if (!__any_sync(0xffffffffu, pending)) break;
    __syncwarp();
  }
  __syncwarp();

}

// Exact MWIS of a window the small-window solver does not take (more than kSmallWindow in-spans, or
// a component with too many leaves).  Out of line like the search path: large and comparatively rare.
__device__ __noinline__ long long stitch_mwis_large(PackedWindowBuf& wb, StitchTables& tb, int E, int nw,
                                                   long long node_limit, int lane) {
  long long nodes = 1;
  __syncwarp();
  if (lane < nw) wb.adj[lane] = window_adjacency(wb, E, nw, lane);
  __syncwarp();
  // lane 0: components one after the other (plain search, Hungarian for E = 1); components
  // whose plain search runs out of budget come back and are searched by the whole warp
  uint32_t deferred[TW_MWIS_MAX_DEFERRED];
  int n_def = 0;
  if (lane == 0) nodes = mwis_solve(wb, E, nw, node_limit, deferred, &n_def);
  nodes = __shfl_sync(0xffffffffu, nodes, 0);
  n_def = __shfl_sync(0xffffffffu, n_def, 0);
  for (int d = 0; d < n_def && nodes >= 0; ++d) {
    const uint32_t comp = __shfl_sync(0xffffffffu, lane == 0 ? deferred[d] : 0u, 0);
    __syncwarp();
    nodes = mwis_component_warp(wb, E, comp, tb.tbl, node_limit, nodes, lane);
  }
  return nodes;
}

__global__ void __launch_bounds__(kStitchWarps * 32, kStitchBlocksPerSM)
k_stitch(tw_batch b, tw_params prm, const uint8_t* __restrict__ cut_all, tw_score_out spec, tw_pass_out out,
         uint32_t* __restrict__ taken, long long node_limit, StitchUnits units, StitchLayout layout,
         StitchTables* __restrict__ tables, int* __restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ double etab[64];
  load_exp_table(etab);
  const int warp_in_block = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // one warp = one UNIT: a stretch [u0, u1) of one service's in-spans that shares no candidate span with
  // the rest of the service (k_stitch_units), or the whole service when no unit list was built
  const int u = blockIdx.x * kStitchWarps + warp_in_block;
  int p, u0 = 0, u1 = -1;
  if (units.prob) {
    if (u >= *units.count) return;
    p = units.prob[u];
    u0 = units.lo[u];
    u1 = units.hi[u];
  } else {
    p = u;
    if (p >= b.n_problems) return;
  }
  const StitchSlab slab{smem_raw + warp_in_block * layout.bytes};
  StitchWarpSmem& sm = slab.fixed();
#ifdef TW_PROFILE_PHASES
  long long _sp_t0 = clock64();
#endif
  int rc = TW_OK;
  if (lane == 0) rc = load_view(b, p, sm.v);
  rc = __shfl_sync(0xffffffffu, rc, 0);
  __syncwarp();
  if (rc != TW_OK) {
    if (lane == 0) { atomicMin(err_flag, rc); if (out.counters) out.counters[p * 4 + 3] = rc; }
    return;
  }
  const ProbView& v = sm.v;
  PackedWindowBuf& wb = slab.window(layout);
  const int n = v.n_in, E = v.E;
  if (u1 < 0) u1 = n;
  const uint8_t* cut = cut_all + v.in_off;

  // taken bitmap of (problem, ep): word-aligned region, see tw_api.cu (taken_words)
  uint32_t* tk_base[TW_MAX_E];
  OutWin w[TW_MAX_E];
  // The taken bitmap lives in this warp's shared memory when the service is small enough (the
  // fast-path test then costs no L2 round trip per window); +2 words of slack per ep because the
  // test reads three consecutive words.
  int tk_words = 0;
  for (int e = 0; e < E; ++e) tk_words += (v.n_out[e] >> 5) + 3;
  const bool tk_smem = tk_words <= layout.tk_words;
  uint32_t* const tk_slab = slab.taken();
  {
    int off = 0;
    for (int e = 0; e < E; ++e) {
      tk_base[e] = tk_smem ? tk_slab + off : taken + (v.out_off[e] >> 5) + (v.ep0 + e);
      off += (v.n_out[e] >> 5) + 3;
      w[e].s = v.os[e]; w[e].e = v.oe[e]; w[e].base = 0; w[e].n = v.n_out[e];
    }
  }
  if (tk_smem)
    for (int x = lane; x < tk_words; x += 32) { tk_slab[x] = 0u; tk_slab[layout.tk_words + x] = 0u; }
  __syncwarp();
  // defaults
  for (int i = u0 + lane; i < u1; i += 32) {
    out.mis_rank[v.in_off + i] = -1;
    for (int e = 0; e < E; ++e) out.assign[v.tuple_off + (int64_t)e * n + i] = -1;
  }
  // the bases param_view(mode, ...) takes in the search tier, as param_view(prm, ...) computes them
  const double* gauss_base = prm.mode == TW_PARAMS_GAUSS_BATCHED
                                 ? prm.gauss + prm.prob_gauss_off[p] * TW_GAUSS_REC : nullptr;
  const double* mix_base = prm.mode == TW_PARAMS_MIXTURE ? prm.mix + (int64_t)v.term0 * TW_MIX_REC : nullptr;

  WindowCursor wc;
  wc.init();
  int not_best = 0, unassigned = 0;
  long long max_nodes = 0;
  int ws = u0;
  bool skip_run = false;
  const bool can_run = tk_smem && spec.used_lo != nullptr && out.topk_score == nullptr;
  TW_SPHASE(0);                                  // setup + defaults
  // The per-in-span records the run / adopt paths read (maps, top-K lists, counts) were written by the
  // scoring kernel and are cold; every step of this sequential walk would otherwise wait for them one
  // dependent miss after the other.  Each lane asks for the records of in-span (ws + 32 + lane) — one
  // warp-width ahead of the step that will read them.
  auto prefetch_ahead = [&](int first) {
    const int ip = first + lane;
    if (spec.used_lo == nullptr || ip >= n) return;
    const int64_t gi = v.in_off + ip;
    const int64_t base = v.tuple_off + (int64_t)ip * E;
    prefetch_l1(spec.used_lo + base);
    prefetch_l1(spec.used_bits + 2 * base);
    prefetch_l1(spec.topk_idx + TW_K * base);
    prefetch_l1(spec.topk_idx + TW_K * base + TW_K * E - 1);
    prefetch_l1(spec.topk_score + gi * TW_K);
    if ((lane & 15) == 0) {
      prefetch_l1(spec.topk_cnt + gi);
      prefetch_l1(spec.used_wide + gi);
      prefetch_l1(spec.n_feasible + gi);
      prefetch_l1(cut + ip);
    }
  };
  prefetch_ahead(u0);
  int prefetched_to = u0 + 32;
  while (ws < u1) {
    if (ws + 32 >= prefetched_to) { prefetch_ahead(prefetched_to); prefetched_to += 32; }
    // ---- run of consecutive ONE-in-span windows, one lane each.  Windows only interact through
    // the taken bits, so if (a) every in-span of the run passes the fast-path test against the bits
    // taken so far and (b) the candidate maps of the run are pairwise disjoint, processing them
    // one after the other would give every one of them its undeleted rank-0 tuple: commit them
    // together.  Anything else falls back to the window-at-a-time path below (same results).
    if (can_run && !skip_run) {
      // a window that starts at ws + j is a single in-span iff the next in-span is a perfect cut
      // (or it is the last one): at a window start the size cap cannot be the reason (count <= 2).
      // After such a run the cursor's count is irrelevant: the next visit sees cut[] set and resets it.
      const int ij = ws + lane;
      const bool single = ij < u1 && (ij == n - 1 ? ij != 0 : cut[ij + 1] != 0);
      const unsigned sm_mask = __ballot_sync(0xffffffffu, single);
      const int R = sm_mask == 0xffffffffu ? 32 : __ffs(~sm_mask) - 1;
      TW_SPHASE(1);                              // run extent (cut flags)
      if (R >= 1) {
        const bool act = lane < R;
        const int ir = ws + (act ? lane : 0);
        const int64_t gi = v.in_off + ir;
        const int64_t base = v.tuple_off + (int64_t)ir * E;
        bool ok = act ? spec.used_wide[gi] == 0 : true;
        if (act && ok) {
          for (int e = 0; e < E; ++e) {
            const int ulo = spec.used_lo[base + e];
            const uint32_t u0 = spec.used_bits[2 * (base + e)], u1 = spec.used_bits[2 * (base + e) + 1];
            if ((u0 | u1) == 0u) continue;
            const int q = ulo >> 5, sh = ulo & 31;
            // the map in the coordinates of the taken bitmap: three words
            const uint32_t m0 = u0 << sh;
            const uint32_t m1 = sh ? (u0 >> (32 - sh)) | (u1 << sh) : u1;
            const uint32_t m2 = sh ? (u1 >> (32 - sh)) : 0u;
            uint32_t* tkp = tk_base[e] + q;
            uint32_t* tmp = tkp + layout.tk_words;
            if ((tkp[0] & m0) | (tkp[1] & m1) | (tkp[2] & m2)) ok = false;          // (a)
            if (m0 && (atomicOr(&tmp[0], m0) & m0)) ok = false;                     // (b)
            if (m1 && (atomicOr(&tmp[1], m1) & m1)) ok = false;
            if (m2 && (atomicOr(&tmp[2], m2) & m2)) ok = false;
          }
        }
        const bool all_ok = __all_sync(0xffffffffu, ok);
        __syncwarp();
        if (act && spec.used_wide[gi] == 0) {   // leave the scratch bitmap zero for the next run
          for (int e = 0; e < E; ++e) {
            const int ulo = spec.used_lo[base + e];
            uint32_t* tmp = tk_base[e] + (ulo >> 5) + layout.tk_words;
            tmp[0] = 0u; tmp[1] = 0u; tmp[2] = 0u;
          }
        }
        __syncwarp();
        TW_SPHASE(2);                            // run test
        if (all_ok) {
          int rank = -2;
          if (act) {
            const int cnt = spec.topk_cnt[gi];
            rank = (cnt > 0 && TW_WEIGHT_OFFSET + spec.topk_score[gi * TW_K] > 0.0) ? 0 : -1;
            out.n_cand[gi] = spec.n_feasible[gi];
            out.mis_rank[gi] = (int8_t)rank;
            if (rank == 0) {
              const int32_t* ix = spec.topk_idx + TW_K * base;
              for (int e = 0; e < E; ++e) {
                const int o = ix[e];
                out.assign[v.tuple_off + (int64_t)e * n + ir] = o;
                atomicOr(&tk_base[e][o >> 5], 1u << (o & 31));
              }
            }
          }
          unassigned += __popc(__ballot_sync(0xffffffffu, act && rank < 0));
          not_best += __popc(__ballot_sync(0xffffffffu, act && rank != 0));
          __syncwarp();
          wc.count = 1;
          ws += R;
          TW_SPHASE(3);                          // run commit
          TW_SCOUNT(10, 1);
          TW_SCOUNT(11, R);
          continue;
        }
        skip_run = true;   // conflict: do this window the long way, then try runs again
      }
    }
    skip_run = false;
    // ---- window extent (uniform across the warp)
    int we = ws;
    {
      // cut[ws .. ws + 63] in registers; a window spans <= 31 in-spans and looks one ahead
      const unsigned c0 = __ballot_sync(0xffffffffu, ws + lane < n && cut[ws + lane] != 0);
      const unsigned c1 = __ballot_sync(0xffffffffu, ws + 32 + lane < n && cut[ws + 32 + lane] != 0);
      const unsigned long long cm = ((unsigned long long)c1 << 32) | c0;
      auto cutbit = [&](int q) { return (int)((cm >> (q - ws)) & 1ull); };
      while (true) {   // WindowCursor::ends_at on the register copy
        bool end;
        if (we == n - 1) end = we != 0;
        else {
          end = false;
          if (we != 0) {
            if (cutbit(we)) wc.count = 0;
            else if (wc.count == TW_MAX_WINDOW) { wc.count = 0; end = true; }
          }
          wc.count += 1;
          if (cutbit(we + 1)) end = true;
        }
        if (end || we >= n - 1) break;
        ++we;
      }
    }
    const int nw = we - ws + 1;
    if (nw > TW_WINDOW_CAP) { rc = TW_ERR_INVALID; break; }
    TW_SPHASE(4);                                // window extent
    TW_SCOUNT(12, 1);
    TW_SCOUNT(13, nw);

    // ---- per-lane candidate ranges on the not-taken spans
    const bool active = lane < nw;
    const int i = ws + (active ? lane : 0);
    const int64_t in_s = v.is[i], in_e = v.ie[i];
    auto is_taken = [&](int e, int o) {   // volatile: bits are set by other lanes with atomics
      return (reinterpret_cast<volatile const uint32_t*>(tk_base[e])[o >> 5] >> (o & 31)) & 1u;
    };
    // ---- fast path: none of the in-span's candidates (the spans of its feasible tuples on the
    // undeleted lists) has been taken => the undeleted top-K list IS FindTopKAssignments(out_copy)
    bool fast = false;
    if (active && spec.used_lo && !spec.used_wide[v.in_off + i]) {
      const int64_t base = v.tuple_off + (int64_t)i * E;
      uint32_t hit = 0;
      for (int e = 0; e < E; ++e) {
        const int ulo = spec.used_lo[base + e];
        const uint32_t u0 = spec.used_bits[2 * (base + e)], u1 = spec.used_bits[2 * (base + e) + 1];
        if ((u0 | u1) == 0u) continue;
        const volatile uint32_t* tkw = reinterpret_cast<volatile const uint32_t*>(tk_base[e]) + (ulo >> 5);
        const int sh = ulo & 31;
        const uint32_t a = tkw[0], bq = tkw[1], c2 = tkw[2];
        hit |= __funnelshift_r(a, bq, sh) & u0;
        hit |= __funnelshift_r(bq, c2, sh) & u1;
      }
      fast = hit == 0u;
    }
    const int batch0 = ws / TW_PARAM_BATCH;
    if (fast) {   // adopt the list computed on the undeleted spans
      const int64_t gi = v.in_off + i;
      const int cnt = spec.topk_cnt[gi];
      out.n_cand[gi] = spec.n_feasible[gi];
      wb.cnt[lane] = cnt;
      const int32_t* ix = spec.topk_idx + TW_K * (v.tuple_off + (int64_t)i * E);
      for (int k = 0; k < cnt; ++k) {
        wb.score[lane][k] = spec.topk_score[gi * TW_K + k];
        for (int e = 0; e < E; ++e) wb.at(lane, k, e) = ix[k * E + e];
      }
      if (out.topk_score) {
        out.topk_cnt[gi] = (uint8_t)cnt;
        int32_t* ox = out.topk_idx + TW_K * (v.tuple_off + (int64_t)i * E);
        for (int k = 0; k < TW_K; ++k) {
          out.topk_score[gi * TW_K + k] = spec.topk_score[gi * TW_K + k];
          for (int e = 0; e < E; ++e) ox[k * E + e] = ix[k * E + e];
        }
      }
    }
    TW_SPHASE(5);                                // fast test + adopt
    // ---- slow path (kept out of line: the hot loop above and below stays small in the instruction cache)
    const unsigned slow_mask = __ballot_sync(0xffffffffu, active && !fast);   // (all lanes vote: the counter macro runs on lane 0 only)
    TW_SCOUNT(14, __popc(slow_mask));
    if (slow_mask)
      stitch_search_lanes(v, wb, tables[u], prm, out, tk_base, w, gauss_base, mix_base, etab, E, lane, ws, i, in_s, in_e,
                          active && !fast, batch0);
    __syncwarp();
    TW_SPHASE(6);                                // slow path
    // ---- stitch the window (V3:1192-1219)
    long long nodes = 1;
    if (nw == 1) {   // one in-span: its best candidate if the vertex weight is positive
      if (lane == 0) wb.chosen[0] = (wb.cnt[0] > 0 && TW_WEIGHT_OFFSET + wb.score[0][0] > 0.0) ? 0 : -1;
    } else {
      bool solved = false;
      if (nw <= kSmallWindow) solved = stitch_small_window(sm, wb, E, nw, lane, &nodes);
      if (!solved) {
        TW_SCOUNT(15, 1);
        nodes = stitch_mwis_large(wb, tables[u], E, nw, node_limit, lane);
      }
    }
    __syncwarp();
    TW_SPHASE(7);                                // adjacency + MWIS
    if (nodes < 0) { rc = TW_ERR_MWIS_LIMIT; break; }
    if (nodes > max_nodes) max_nodes = nodes;
    int rank = -2;
    if (lane < nw) {
      rank = wb.chosen[lane];
      out.mis_rank[v.in_off + i] = (int8_t)rank;
      if (rank >= 0) {
        for (int e = 0; e < E; ++e) {
          int o = wb.at(lane, rank, e);
          out.assign[v.tuple_off + (int64_t)e * n + i] = o;
          atomicOr(&tk_base[e][o >> 5], 1u << (o & 31));
        }
      }
    }
    not_best += __popc(__ballot_sync(0xffffffffu, lane < nw && rank != 0));
    unassigned += __popc(__ballot_sync(0xffffffffu, lane < nw && rank < 0));
    if (!tk_smem) __threadfence_block();
    __syncwarp();
    ws = we + 1;
    TW_SPHASE(8);                                // window commit
  }
  if (lane == 0) {
    if (rc != TW_OK) atomicMin(err_flag, rc);
    if (out.counters) {          // zeroed by launch_stitch; several units of one service add up
      atomicAdd(&out.counters[p * 4 + 0], not_best);
      atomicAdd(&out.counters[p * 4 + 1], unassigned);
      atomicMax(&out.counters[p * 4 + 2], (int)(max_nodes > 0x7fffffffLL ? 0x7fffffffLL : max_nodes));
      atomicMin(&out.counters[p * 4 + 3], rc);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Units of the stitch: intra-service parallelism.  The hot loop of the reference is one sequential
// walk per service, but only because deletion couples windows that compete for the same spans.  A
// perfect cut at in-span i is STRONG when, for every callee, every candidate position of the in-spans
// before i lies below the first position an in-span from i on can use (lists and in-spans are sorted by
// start, so that first position, lower_bound(in_i.start), is a lower bound for all later in-spans too).
// Candidates with deletion are a subset of the candidates on the undeleted lists (the maps of the
// scoring kernel), so the two sides of a strong cut never read or take the same span: they can be
// stitched by different warps in any order with the result of the sequential walk.  One warp per
// service scans its in-spans 32 at a time (exclusive prefix maximum of the highest candidate position
// per callee) and closes a unit at a strong cut once it holds at least `min_len` in-spans.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_stitch_units(tw_batch b, const uint8_t* __restrict__ cut_all, tw_score_out spec, int min_len, StitchUnits units) {
  const int p = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= b.n_problems) return;
  const int ep0 = b.prob_ep_off[p], E = b.prob_ep_off[p + 1] - ep0;
  const int64_t in_off = b.prob_in_off[p];
  const int n = (int)(b.prob_in_off[p + 1] - in_off);
  const int64_t tuple_off = b.prob_tuple_off[p];
  const uint8_t* cut = cut_all + in_off;
  int run_max[TW_MAX_E];
#pragma unroll
  for (int e = 0; e < TW_MAX_E; ++e) run_max[e] = -1;
  int unit_start = 0;
  auto emit = [&](int a, int z) {
    if (lane == 0) {
      const int idx = atomicAdd(units.count, 1);
      units.prob[idx] = p;
      units.lo[idx] = a;
      units.hi[idx] = z;
    }
  };
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    const bool valid = i < n;
    bool strong = valid && i >= 1 && cut[i] != 0;
    const int64_t gi = in_off + i;
    const bool wide = valid ? spec.used_wide[gi] != 0 : false;
#pragma unroll
    for (int e = 0; e < TW_MAX_E; ++e) {
      if (e >= E) break;
      int first = 0x7fffffff, hi = -1;
      if (valid) {
        const int64_t off = b.ep_out_off[ep0 + e];
        const int no = (int)(b.ep_out_off[ep0 + e + 1] - off);
        if (wide) {
          first = lower_bound(b.out_start + off, no, b.in_start[gi]);
          hi = upper_bound(b.out_start + off, no, b.in_end[gi]) - 1;
        } else {
          const int64_t q = tuple_off + (int64_t)i * E + e;
          first = spec.used_lo[q];
          const uint32_t m0 = spec.used_bits[2 * q], m1 = spec.used_bits[2 * q + 1];
          hi = m1 ? first + 63 - __clz(m1) : m0 ? first + 31 - __clz(m0) : -1;
        }
      }
      // exclusive prefix maximum of hi over the lanes, seeded with the maximum of the earlier chunks
      int pm = hi;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, pm, d);
        if (lane >= d) pm = o > pm ? o : pm;
      }
      int ex = __shfl_up_sync(0xffffffffu, pm, 1);
      if (lane == 0) ex = -1;
      ex = ex > run_max[e] ? ex : run_max[e];
      if (!(ex < first)) strong = false;
      const int tot = __shfl_sync(0xffffffffu, pm, 31);
      run_max[e] = tot > run_max[e] ? tot : run_max[e];
    }
    unsigned sm = __ballot_sync(0xffffffffu, strong);
    while (sm) {
      const int q = base + __ffs(sm) - 1;
      sm &= sm - 1u;
      if (q - unit_start >= min_len) { emit(unit_start, q); unit_start = q; }
    }
  }
  emit(unit_start, n);
}

#ifdef TW_PROFILE_PHASES
extern "C" int tw_debug_stitch_phases(unsigned long long* out16, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out16, g_stitch_phase, sizeof(unsigned long long) * 16);
  if (e != cudaSuccess) return -2;
  if (reset) {
    unsigned long long z[16] = {0};
    cudaMemcpyToSymbol(g_stitch_phase, z, sizeof z);
  }
  return 0;
}
#endif

StitchLayout stitch_layout(int e_max, int tk_words_max) {
  StitchLayout L;
  L.tk_words = tk_words_max < kTakenWords ? tk_words_max : kTakenWords;
  L.wb_off = (int)sizeof(StitchWarpSmem) + 2 * L.tk_words * (int)sizeof(uint32_t);
  L.bytes = (L.wb_off + PackedWindowBuf::packed_bytes(e_max) + 15) & ~15;
  return L;
}

cudaError_t setup_stitch() {   // the largest slab any batch can ask for
  return cudaFuncSetAttribute(k_stitch, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              stitch_layout(TW_MAX_E, kTakenWords).bytes * kStitchWarps);
}

cudaError_t launch_stitch(const tw_batch& b, const tw_params& prm, const uint8_t* cut,
                          const tw_score_out& spec, const tw_pass_out& out, uint32_t* taken_words, size_t taken_n_words,
                          long long node_limit, const StitchUnits& unit_buf, int max_units, const StitchLayout& layout,
                          StitchTables* tables, int* err_flag, cudaStream_t s, int64_t& launches) {
  cudaError_t e = cudaMemsetAsync(taken_words, 0, taken_n_words * sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  if (out.counters) {
    e = cudaMemsetAsync(out.counters, 0, (size_t)b.n_problems * 4 * sizeof(int32_t), s);
    if (e != cudaSuccess) return e;
  }
  const size_t smem = (size_t)layout.bytes * kStitchWarps;
  StitchUnits units{nullptr, nullptr, nullptr, nullptr};
  int warps = b.n_problems;
  // Units pay when services alone cannot fill the machine (a shipped directory has 2-6 services; the
  // 132 SMs of an H100 hold ~2500 stitch warps); with thousands of services one warp per service is
  // already enough parallelism and the unit pre-pass + per-unit set-up cost more than the shorter tail
  // gains.  The maps of the scoring kernel prove which cuts are strong.
  if (spec.used_lo && unit_buf.prob && max_units > 0 && b.n_problems < kStitchUnitMaxServices) {
    units = unit_buf;
    e = cudaMemsetAsync(units.count, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    k_stitch_units<<<(b.n_problems + 3) / 4, 128, 0, s>>>(b, cut, spec, kStitchUnitMin, units);
    e = after_launch(launches);
    if (e != cudaSuccess) return e;
    warps = max_units;
  }
  int blocks = (warps + kStitchWarps - 1) / kStitchWarps;
  k_stitch<<<blocks, kStitchWarps * 32, smem, s>>>(b, prm, cut, spec, out, taken_words, node_limit, units, layout,
                                                   tables, err_flag);
  return after_launch(launches);
}

}  // namespace tw
