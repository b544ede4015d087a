// tw_emul.cpp — CPU stepping of the engine's per-thread device functions (tw_core.cuh).
//
// TEST INFRASTRUCTURE ONLY, for machines without a GPU: logic errors are caught by `pytest -m "not gpu"`
// before a GPU run is spent.  It is not linked into libtw_b200.so and the package never loads it: the
// product has no CPU path.
//
// The device functions themselves, compiled here with g++ from the headers the kernels include:
// load_view, param_view, term_logpdf / score_tuple, enumerate, the term tables (term_table_* ,
// table_score, enumerate_combos), the top-K list (topk_offer, topk_offer_sorted, topk_finish,
// store_topk_row), bitmaps_intersect, WindowCursor, window_adjacency, mwis_solve, assignment_solve,
// the small-window search (small_component, small_strides, small_leaf, SmallBest::offer / merge,
// small_decode), assess_in_span, and the whole skip regime of tw_skip_core.cuh.
//
// Orchestration written for the CPU, mirroring tw_score.cu (k_score), tw_stitch.cu (k_stitch),
// tw_assess.cu (k_assess), tw_skip.cu (k_skip) and tw_skip_assess.cu (k_skip_assess) but not shared
// with them: the loops over threads, lanes and butterfly steps; the prev-index scan and the cut flags
// of twe_score_problem; the K + 1 head-merge rounds of the heavy-in-span path in enumerate_with_tables
// (ballots and shuffles in the kernels); the conflict masks of twe_small_window (__match_any_sync in
// the kernel); the taken bitmap as a byte array.  The kernels' tiers that only choose where a list
// comes from (run / adopt in k_stitch, the work-balanced k_score3) have no counterpart here.
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../traceweaver_b200/csrc/tw_core.cuh"

using namespace tw;

// Two knobs of twe_score_problem / twe_stitch_problem select the kernels' code paths:
//   table_cap     term-table slots available per in-span (shared memory in the kernels); in-spans whose
//                 tables do not fit take the lazy per-leaf path, so 0 forces it.
//   light_combos  in-spans with more candidate combinations go through the lane-parallel path (32 lanes
//                 stride over the combos, partial top-K lists are merged); -1 disables it.  As in step 1
//                 of warp_topk_search (tw_score.cu) and its copy in the stitch, an equal score or a NaN
//                 among the six best sends the in-span back to the sequential heap replay.

// one in-span through the table path: fill -> evaluate every slot -> DFS with look-ups
template <class Taken>
static long long enumerate_with_tables(const ProbView& v, const ParamView& pv, int64_t in_s, int64_t in_e,
                                       const OutWin* w, const int* lo, const int* r, int table_size, Taken taken,
                                       TopK& tk, uint32_t* mark, int W, int* overflow, long long light_combos) {
  std::vector<double> tbl((size_t)table_size + 1);
  std::vector<uint8_t> sid((size_t)table_size + 1);
  int o_last[TW_MAX_E], lo_abs[TW_MAX_E];
  term_table_last_offsets(v, r, o_last);
  for (int e = 0; e < v.E; ++e) lo_abs[e] = w[e].base + lo[e];
  term_table_fill(v, in_s, in_e, w, lo, r, o_last, 0, taken, tbl.data(), sid.data());
  for (int s = 0; s < table_size; ++s)              // the dense, lane-parallel pass of the kernels
    if (sid[s] != TW_SLOT_INVALID) tbl[s] = term_logpdf(pv, sid[s] & 63, tbl[s]);
  long long leaves = 0;
  const long long P = combo_count(v, r);
  if (light_combos >= 0 && P > light_combos && P < (1LL << 40)) {
    const int L = 32;
    std::vector<TopK> part(L);
    bool tie = false;
    for (int lane = 0; lane < L; ++lane) {
      part[lane].n = 0;
      enumerate_combos(v, w, lo, r, o_last, sid.data(), lane, L, P,
                       [&](const int* c, const int64_t* ce, long long) {
                         ++leaves;
                         if (mark)
                           for (int e = 0; e < v.E; ++e) {
                             int bit = c[e] - lo_abs[e];
                             if (bit >= 32 * W) { *overflow = 1; continue; }
                             mark[e * W + (bit >> 5)] |= 1u << (bit & 31);
                           }
                         const double sc = table_score(v, r, lo_abs, tbl.data(), c, ce);
                         for (int k = 0; k < part[lane].n; ++k) tie = tie || part[lane].score[k] == sc;
                         tie = tie || sc != sc;
                         topk_offer_sorted(v, part[lane], sc, c);
                       });
    }
    // K + 1 rounds of "best head over the lanes": a maximum held by two lanes, or equal to the previous
    // round's, is a tie among the six best
    int head[32] = {0};
    double prev = 0.0;
    for (int round = 0; round <= TW_K; ++round) {
      double mx = -INFINITY;
      for (int lane = 0; lane < L; ++lane)
        if (head[lane] < part[lane].n && part[lane].score[head[lane]] > mx) mx = part[lane].score[head[lane]];
      if (!(mx > -INFINITY)) break;
      int best = -1, holders = 0;
      for (int lane = 0; lane < L; ++lane)
        if (head[lane] < part[lane].n && part[lane].score[head[lane]] == mx) {
          if (best < 0) best = lane;
          ++holders;
        }
      if (holders > 1 || (round > 0 && mx == prev)) tie = true;
      prev = mx;
      if (round < TW_K) {
        tk.score[tk.n] = mx;
        for (int e = 0; e < v.E; ++e) tk.idx[tk.n][e] = part[best].idx[head[best]][e];
        ++tk.n;
      }
      ++head[best];
    }
    if (!tie) return leaves;
    tk.clear();                            // the owner redoes the in-span alone (step 2)
    leaves = 0;
  }
  enumerate(v, in_s, in_e, w, lo,
            [&](int e, int o) { return sid[o_last[e] + (o - lo_abs[e])] == TW_SLOT_INVALID; },
            [&](const int* c, const int64_t*, const int64_t* ce) {
              ++leaves;
              if (mark)
                for (int e = 0; e < v.E; ++e) {
                  int bit = c[e] - lo_abs[e];
                  if (bit >= 32 * W) { *overflow = 1; continue; }
                  mark[e * W + (bit >> 5)] |= 1u << (bit & 31);
                }
              topk_offer(v, tk, table_score(v, r, lo_abs, tbl.data(), c, ce), c);
            });
  return leaves;
}

extern "C" int twe_score_problem(const tw_batch* b, int p, const tw_params* prm, const tw_score_out* out,
                                 int W, int* overflow, int table_cap, long long light_combos) {
  ProbView v;
  int rc = load_view(*b, p, v);
  if (rc) return rc;
  int n = v.n_in;
  // exclusive prefix arg-max of in_end, ties to the later index (k_prev_index)
  std::vector<int> prev(n, 0);
  for (int i = 1; i < n; ++i) {
    int pr = prev[i - 1];
    if (i >= 2 && v.ie[i - 1] >= v.ie[pr]) pr = i - 1;
    if (i == 1) pr = 0;
    prev[i] = pr;
  }
  std::vector<uint32_t> used((size_t)n * TW_MAX_E * W, 0u);
  std::vector<int> lo_abs((size_t)n * TW_MAX_E, 0);
  OutWin w[TW_MAX_E];
  for (int e = 0; e < v.E; ++e) w[e] = OutWin{v.os[e], v.oe[e], 0, v.n_out[e]};
  *overflow = 0;
  for (int i = 0; i < n; ++i) {
    int lo[TW_MAX_E];
    for (int e = 0; e < v.E; ++e) {
      lo[e] = lower_bound(w[e].s, w[e].n, v.is[i]);
      lo_abs[(size_t)i * TW_MAX_E + e] = lo[e];
    }
    TopK tk; tk.clear();
    long long leaves = 0;
    uint32_t* mine = &used[(size_t)i * TW_MAX_E * W];
    ParamView pv;
    if (prm) pv = param_view(*prm, v, p, i / TW_PARAM_BATCH, nullptr);
    int64_t in_s = v.is[i], in_e = v.ie[i];
    int r[TW_MAX_E];
    for (int e = 0; e < v.E; ++e) r[e] = range_len(w[e], lo[e], in_e);
    int tsize = term_table_size(v, r);
    if (prm && tsize <= table_cap) {
      leaves = enumerate_with_tables(v, pv, in_s, in_e, w, lo, r, tsize, [](int, int) { return false; }, tk, mine,
                                     W, overflow, light_combos);
    } else {
      enumerate(v, in_s, in_e, w, lo, [](int, int) { return false; },
                [&](const int* c, const int64_t* cs, const int64_t* ce) {
                  ++leaves;
                  for (int e = 0; e < v.E; ++e) {
                    int bit = c[e] - lo[e];
                    if (bit >= 32 * W) { *overflow = 1; continue; }
                    mine[e * W + (bit >> 5)] |= 1u << (bit & 31);
                  }
                  if (prm) topk_offer(v, tk, score_tuple(v, pv, in_s, in_e, cs, ce), c);
                });
    }
    topk_finish(v, tk);
    out->n_feasible[v.in_off + i] = (int32_t)leaves;
    if (prm && out->topk_score)
      store_topk_row(tk, v.E, out->topk_score + (v.in_off + i) * TW_K,
                     out->topk_idx + TW_K * (v.tuple_off + (int64_t)i * v.E), out->topk_cnt + v.in_off + i);
  }
  for (int i = 0; i < n; ++i) {
    uint8_t cut = 0;
    if (i >= 1 && i <= n - 2) {
      int pi = prev[i];
      bool disjoint = true;
      for (int e = 0; e < v.E && disjoint; ++e)
        if (bitmaps_intersect(&used[((size_t)pi * TW_MAX_E + e) * W], lo_abs[(size_t)pi * TW_MAX_E + e],
                              &used[((size_t)i * TW_MAX_E + e) * W], lo_abs[(size_t)i * TW_MAX_E + e], W))
          disjoint = false;
      cut = (uint8_t)(disjoint && v.ie[pi] <= v.ie[i]);
    }
    out->cut[v.in_off + i] = cut;
  }
  return TW_OK;
}

extern "C" int twe_stitch_problem(const tw_batch* b, int p, const tw_params* prm, const uint8_t* cut_all,
                                  const tw_pass_out* out, long long node_limit, int table_cap,
                                  long long light_combos) {
  ProbView v;
  int rc = load_view(*b, p, v);
  if (rc) return rc;
  int n = v.n_in;
  const uint8_t* cut = cut_all + v.in_off;
  std::vector<std::vector<uint8_t>> taken(v.E);
  for (int e = 0; e < v.E; ++e) taken[e].assign((size_t)v.n_out[e], 0);
  OutWin w[TW_MAX_E];
  for (int e = 0; e < v.E; ++e) w[e] = OutWin{v.os[e], v.oe[e], 0, v.n_out[e]};
  for (int e = 0; e < v.E; ++e)
    for (int i = 0; i < n; ++i) out->assign[v.tuple_off + (int64_t)e * n + i] = -1;
  for (int i = 0; i < n; ++i) out->mis_rank[v.in_off + i] = -1;
  WindowCursor wc; wc.init();
  WindowBuf* wb = new WindowBuf;
  int cursor[TW_MAX_E] = {0};
  int not_best = 0, unassigned = 0; long long max_nodes = 0;
  int ws = 0;
  while (ws < n) {
    int we = ws;
    while (!wc.ends_at(we, n, cut) && we < n - 1) ++we;
    bool closes = (we != n - 1) || (n > 1);
    int nw = we - ws + 1;
    if (nw > TW_WINDOW_CAP) { delete wb; return TW_ERR_INVALID; }
    for (int l = 0; l < nw; ++l) {  // one lane per in-span of the window
      int i = ws + l;
      int lo[TW_MAX_E];
      for (int e = 0; e < v.E; ++e) lo[e] = lower_bound_from(w[e].s, w[e].n, cursor[e], v.is[i]);
      if (l == 0) for (int e = 0; e < v.E; ++e) cursor[e] = lo[e];
      TopK tk; tk.clear();
      long long leaves = 0;
      const ParamView pv = param_view(*prm, v, p, i / TW_PARAM_BATCH, nullptr);
      int64_t in_s = v.is[i], in_e = v.ie[i];
      int r[TW_MAX_E];
      for (int e = 0; e < v.E; ++e) r[e] = range_len(w[e], lo[e], in_e);
      int tsize = term_table_size(v, r);
      auto is_taken = [&](int e, int o) { return taken[e][o] != 0; };
      if (tsize <= table_cap) {
        int ov = 0;
        leaves = enumerate_with_tables(v, pv, in_s, in_e, w, lo, r, tsize, is_taken, tk, nullptr, 0, &ov,
                                       light_combos);
      } else {
        enumerate(v, in_s, in_e, w, lo, is_taken,
                  [&](const int* c, const int64_t* cs, const int64_t* ce) {
                    ++leaves;
                    topk_offer(v, tk, score_tuple(v, pv, in_s, in_e, cs, ce), c);
                  });
      }
      topk_finish(v, tk);
      out->n_cand[v.in_off + i] = (int32_t)leaves;
      wb->cnt[l] = tk.n;
      for (int k = 0; k < tk.n; ++k) {
        wb->score[l][k] = tk.score[k];
        for (int e = 0; e < v.E; ++e) wb->idx[l][k][e] = tk.idx[k][e];
      }
      if (out->topk_score)
        store_topk_row(tk, v.E, out->topk_score + (v.in_off + i) * TW_K,
                       out->topk_idx + TW_K * (v.tuple_off + (int64_t)i * v.E), out->topk_cnt + v.in_off + i);
    }
    if (closes) {
      for (int l = 0; l < nw; ++l) wb->adj[l] = window_adjacency(*wb, v.E, nw, l);
      long long nodes = mwis_solve(*wb, v.E, nw, node_limit);
      if (nodes < 0) { delete wb; return TW_ERR_MWIS_LIMIT; }
      if (nodes > max_nodes) max_nodes = nodes;
      for (int l = 0; l < nw; ++l) {
        int i = ws + l, r = wb->chosen[l];
        out->mis_rank[v.in_off + i] = (int8_t)r;
        if (r != 0) ++not_best;
        if (r < 0) { ++unassigned; continue; }
        for (int e = 0; e < v.E; ++e) {
          int o = wb->idx[l][r][e];
          out->assign[v.tuple_off + (int64_t)e * n + i] = o;
          taken[e][o] = 1;
        }
      }
    }
    ws = we + 1;
  }
  if (out->counters) {
    out->counters[p * 4 + 0] = not_best;
    out->counters[p * 4 + 1] = unassigned;
    out->counters[p * 4 + 2] = (int32_t)(max_nodes > 0x7fffffff ? 0x7fffffff : max_nodes);
    out->counters[p * 4 + 3] = 0;
  }
  delete wb;
  return TW_OK;
}

static double butterfly32(double* x) {
  for (int d = 16; d > 0; d >>= 1) {
    double y[32];
    for (int l = 0; l < 32; ++l) y[l] = dadd(x[l], x[l ^ d]);
    for (int l = 0; l < 32; ++l) x[l] = y[l];
  }
  return x[0];
}

// k_assess / k_skip_assess for one problem: assess_one(i, gi) per in-span (thread), the tile partials and
// their per-service sum in the kernels' order (butterfly over 32 lanes, warps in order, then tile
// partials strided over 32 lanes and a butterfly).  NC: the code count; `margin` may be NULL.
template <int NC, class AssessOne>
static void step_assess(const ProbView& v, int p, AssessOne assess_one, double* score, uint8_t* code,
                        double* margin, double* prob_sum, int32_t* prob_count) {
  const int n_tiles = (v.n_in + 127) / 128;
  std::vector<double> tile_sum((size_t)n_tiles);
  for (int q = 0; q < NC; ++q) prob_count[(size_t)p * NC + q] = 0;
  for (int t = 0; t < n_tiles; ++t) {
    double wsum[4];
    for (int w = 0; w < 4; ++w) {
      double lanes[32];
      for (int l = 0; l < 32; ++l) {
        const int i = t * 128 + w * 32 + l;
        lanes[l] = 0.0;
        if (i >= v.n_in) continue;
        const int64_t gi = v.in_off + i;
        const Assessment a = assess_one(i, gi);
        score[gi] = a.score;
        code[gi] = (uint8_t)a.code;
        if (margin) margin[gi] = a.margin;
        prob_count[(size_t)p * NC + a.code] += 1;
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
}

// k_assess (tw_assess.cu): assess_in_span per in-span; `top` (a final top-K) may be NULL (no margin)
extern "C" int twe_assess_problem(const tw_batch* b, int p, const tw_params* prm, const int32_t* assign,
                                  const tw_score_out* top, double* score, uint8_t* code, double* margin,
                                  double* prob_sum, int32_t* prob_count) {
  ProbView v;
  int rc = load_view(*b, p, v);
  if (rc) return rc;
  step_assess<TW_ASSESS_NCODES>(
      v, p,
      [&](int i, int64_t gi) {
        return assess_in_span(v, param_view(*prm, v, p, i / TW_PARAM_BATCH, nullptr), i, assign, top ? top->topk_score + gi * TW_K : nullptr,
                              top ? top->topk_idx + TW_K * (v.tuple_off + (int64_t)i * v.E) : nullptr,
                              top ? top->topk_cnt[gi] : 0);
      },
      score, code, top ? margin : nullptr, prob_sum, prob_count);
  return TW_OK;
}

// exact matching of one E = 1 window given as candidate lists (unit test against scipy)
extern "C" int twe_assign_window(int nw, const int* cnt, const double* score, const int* span, int* chosen) {
  WindowBuf* wb = new WindowBuf;
  int member[TW_WINDOW_CAP];
  for (int k = 0; k < nw; ++k) {
    wb->cnt[k] = cnt[k];
    member[k] = k;
    for (int r = 0; r < cnt[k]; ++r) { wb->score[k][r] = score[k * TW_K + r]; wb->idx[k][r][0] = span[k * TW_K + r]; }
  }
  assignment_solve(*wb, member, nw, 0, chosen, nullptr, nullptr);
  delete wb;
  return 0;
}

// one window through the sequential solver of the stitch kernel (adjacency + components + branch and
// bound / Hungarian); returns the node count (-1 = node limit)
extern "C" long long twe_mwis_window(int nw, int E, const int* cnt, const double* score, const int* idx,
                                     int* chosen, long long node_limit) {
  WindowBuf* wb = new WindowBuf;
  for (int k = 0; k < nw; ++k) {
    wb->cnt[k] = cnt[k];
    for (int r = 0; r < cnt[k]; ++r) {
      wb->score[k][r] = score[k * TW_K + r];
      for (int e = 0; e < E; ++e) wb->idx[k][r][e] = idx[(k * TW_K + r) * E + e];
    }
  }
  for (int k = 0; k < nw; ++k) wb->adj[k] = window_adjacency(*wb, E, nw, k);
  long long nodes = mwis_solve(*wb, E, nw, node_limit);
  for (int k = 0; k < nw; ++k) chosen[k] = wb->chosen[k];
  delete wb;
  return nodes;
}

// stitch_small_window (tw_stitch.cu) stepped lane by lane: the component search, the leaves, each lane's
// running best and the merge of the lanes are the kernel's own functions (tw_core.cuh, small_component
// .. SmallBest).  Written out here: what the kernel gets from warp collectives — the validity ballot,
// the conflict masks of __match_any_sync, the atomicOr into the in-span adjacency — and the loops over
// the 32 lanes and the five butterfly steps.  Returns 0 when the kernel would fall back to the
// sequential solver (E == 1 component of >= 3 in-spans, or more than `space_cap` leaves).
extern "C" int twe_small_window(int nw, int E, const int* cnt_in, const double* score, const int* idx,
                                int* chosen, int space_cap) {
  if (nw > kSmallWindow) return 0;
  uint32_t cconf[32] = {0};
  double cw[32] = {0};
  int cnt[kSmallWindow];
  uint32_t adj[kSmallWindow] = {0};
  for (int a = 0; a < kSmallWindow; ++a) cnt[a] = a < nw ? cnt_in[a] : 0;
  auto valid = [&](int lane) { return lane / TW_K < nw && lane % TW_K < cnt_in[lane / TW_K]; };
  for (int lane = 0; lane < 32; ++lane) {
    if (!valid(lane)) continue;
    cw[lane] = TW_WEIGHT_OFFSET + score[lane];
    for (int o = 0; o < 32; ++o) {
      if (!valid(o) || o / TW_K == lane / TW_K) continue;
      for (int e = 0; e < E; ++e)
        if (idx[lane * E + e] == idx[o * E + e]) cconf[lane] |= 1u << o;
    }
    for (int a = 0; a < kSmallWindow; ++a)
      if ((cconf[lane] >> (TW_K * a)) & 0x1fu) adj[lane / TW_K] |= 1u << a;
  }
  for (int k = 0; k < nw; ++k) chosen[k] = -1;
  uint32_t todo = (1u << nw) - 1u;
  while (todo) {
    const int seed = lowest_bit(todo);
    const uint32_t comp = small_component(adj, seed);
    todo &= ~comp;
    const int m = __builtin_popcount(comp);
    if (m == 1) {
      if (cnt[seed] > 0 && cw[TW_K * seed] > 0.0) chosen[seed] = 0;
      continue;
    }
    if (E == 1 && m >= 3) return 0;
    int stride[kSmallWindow];
    const int space = small_strides(comp, cnt, stride);
    if (space > space_cap) return 0;
    SmallBest best[32];
    for (int lane = 0; lane < 32; ++lane)
      for (int leaf = lane; leaf < space; leaf += 32) {
        double tot;
        if (small_leaf(comp, cnt, stride, cw, cconf, leaf, &tot)) best[lane].offer(tot, leaf);
      }
    for (int d = 16; d > 0; d >>= 1) {
      SmallBest before[32];
      for (int lane = 0; lane < 32; ++lane) before[lane] = best[lane];
      for (int lane = 0; lane < 32; ++lane) best[lane].merge(before[lane ^ d]);
    }
    small_decode(comp, cnt, stride, best[0].idx, [&](int a, int rank) { chosen[a] = rank; });
  }
  return 1;
}

// ---------------------------------------------------------------------------------------------
// skip / cache mode (tw_skip_core.cuh): the kernel body of k_skip and k_build_dist on the CPU
// ---------------------------------------------------------------------------------------------
#include "../../traceweaver_b200/csrc/tw_skip_core.cuh"

extern "C" int twe_skip_solve(const tw_batch* b, const tw_skip_desc* sd, const tw_skip_out* out, long long node_limit) {
  const int P = b->n_problems;
  std::vector<int64_t> set_off((size_t)P + 1, 0);
  for (int p = 0; p < P; ++p) {
    int64_t words = 0;
    for (int ep = b->prob_ep_off[p]; ep < b->prob_ep_off[p + 1]; ++ep)
      words += (b->ep_out_off[ep + 1] - b->ep_out_off[ep] + 31) / 32;
    set_off[p + 1] = set_off[p] + words;
  }
  std::vector<uint32_t> sets((size_t)(3 * set_off[P]) + 1), taken((size_t)(b->n_out_total / 32) + (size_t)b->n_ep_total + 2);
  std::vector<int32_t> win((size_t)(2 * sd->prob_cnt_off[P]) + 1);
  int rc = TW_OK;
  SkipShared* sh = new SkipShared;
  for (int p = 0; p < P; ++p) {
    const int r = skip_solve_problem(*b, p, *sd, *out, taken.data(), sets.data(), set_off.data(), win.data(), node_limit, *sh);
    if (r < rc) rc = r;
  }
  delete sh;
  return rc;
}

// k_skip_assess (tw_skip_assess.cu): skip_assess_in_span per in-span; `top2` may be NULL (no margin)
extern "C" int twe_skip_assess_problem(const tw_batch* b, int p, const tw_skip_desc* sd, const int32_t* assign,
                                       const tw_skip_out* top2, double* score, uint8_t* code, double* margin,
                                       double* prob_sum, int32_t* prob_count) {
  ProbView v;
  int rc = load_view(*b, p, v);
  if (rc) return rc;
  const SkipProb sp = skip_prob(*sd, v, p);
  step_assess<TW_SKIP_ASSESS_NCODES>(
      v, p,
      [&](int i, int64_t gi) {
        return skip_assess_in_span(v, sp, i, assign, top2 ? top2->top2_score + gi * TW_K : nullptr,
                                   top2 ? top2->top2_idx + TW_K * (v.tuple_off + (int64_t)i * v.E) : nullptr,
                                   top2 ? top2->top2_cnt[gi] : 0);
      },
      score, code, top2 ? margin : nullptr, prob_sum, prob_count);
  return TW_OK;
}

// first_centre (the refit's first k-means++ centre) of every (u[i], n[i])
extern "C" void twe_first_centre(int64_t m, const double* u, const int32_t* n, int32_t* out) {
  for (int64_t i = 0; i < m; ++i) out[i] = first_centre(u[i], n[i]);
}
