// tw_skip_core.cuh — per-thread logic of the skip / cache mode (see tw_skip.cu for what it replaces).
// `__host__ __device__` like tw_core.cuh, so tests/emul steps the very same code on the CPU.
#pragma once
#include "tw_core.cuh"

namespace tw {

constexpr int kSkipCand = 96;                    // candidates of one ep inside one in-span
constexpr int kSkipTouched = 384;                // bitmap words a candidate set may touch before it is cleared wholesale
constexpr double kSqrt2Pi = 2.5066282746310002;  // scipy _norm_pdf_C = sqrt(2 pi)
constexpr double kLogSqrt2Pi = 0.91893853320467274178;   // _norm_pdf_logC
constexpr double kFixedScale = 4398046511104.0;  // 2^42: weights in [2^10, 2^14) are integers at this scale

struct SkipProb {
  int n_win;
  const int64_t* win_start;      // sorted (FetchSkipFromWindow sorts before every look-up, V3:830)
  const int32_t* skip_count;     // [E][n_win]
  int32_t* skip_base;            // [E][n_win] exclusive prefix of skip_count over the windows
  int32_t* fetches;              // [E][n_win]
  const double* pair;            // [(E+1)^2][2]
  int normalized;
  const int8_t* pred_order;      // [E][TW_MAX_E]
  const int32_t* entry_pos[TW_MAX_E];
  const int32_t* sorted_of_entry[TW_MAX_E];
};

// The model and lists of problem p as tw_skip_desc describes them.  skip_base / fetches, the search's
// per-window cursors, are scratch of the caller that searches; they stay NULL here.
TW_HD SkipProb skip_prob(const tw_skip_desc& sd, const ProbView& v, int p) {
  SkipProb sp;
  sp.n_win = (int)(sd.prob_win_off[p + 1] - sd.prob_win_off[p]);
  sp.win_start = sd.win_start + sd.prob_win_off[p];
  sp.skip_count = sd.skip_count + sd.prob_cnt_off[p];
  sp.skip_base = nullptr;
  sp.fetches = nullptr;
  sp.pair = sd.pair_gauss + 2 * sd.prob_pair_off[p];
  sp.normalized = sd.prob_normalized[p];
  sp.pred_order = sd.ep_pred_order + (size_t)v.ep0 * TW_MAX_E;
  for (int e = 0; e < v.E; ++e) {
    sp.entry_pos[e] = sd.out_entry_pos + v.out_off[e];
    sp.sorted_of_entry[e] = sd.out_sorted_of_entry + v.out_off[e];
  }
  return sp;
}

struct SkipShared {
  WindowBuf wb;
  TopK tk;
  int cand[TW_MAX_E][kSkipCand];
  int ncand[TW_MAX_E];
  int touched[3][kSkipTouched];
  int ntouched[3];
  int win_member[TW_WINDOW_CAP];
};

TW_HD void raise(int* err_flag, int code) { if (code < *err_flag) *err_flag = code; }   // err_flag: the caller's local status word

// GetEpPairCost, V1:117-139, for the (mean, std) tuples BuildDistributions leaves in services_times
TW_HD_NOINLINE inline double pair_cost(const SkipProb& sp, int E, int a, int b, int64_t dt, bool* undefined) {
  const double* rec = sp.pair + 2 * (a * (E + 1) + b);
  const double mean = rec[0];
  double sd = rec[1];
  if (mean != mean) { *undefined = true; return 0.0; }     // KeyError in the reference
  if (sd < 1.0e-12) sd = 0.001;
  const double y = ddiv(dsub((double)dt, mean), sd);
  const double h = ddiv(-dmul(y, y), 2.0);
  if (sp.normalized) return ddiv(ddiv(exp(h), kSqrt2Pi), sd);          // scipy.stats.norm.pdf
  return dsub(dsub(h, kLogSqrt2Pi), log(sd));                          // scipy.stats.norm.logpdf
}

TW_HD_NOINLINE inline bool edge_primary(const ProbView& v, int b, int e) {   // AlsoNonPrimaryAncestor, V1:294-303
  for (int x = 0; x < v.E; ++x)
    if (x != b && x != e && (v.pred[x] >> b & 1u) && (v.pred[e] >> x & 1u)) return false;
  return true;
}

// ScoreAssignmentAsPerInvocationGraph, V1:305-361; c[e] >= 0: index into the (sorted) list, < 0: skip span
TW_HD_NOINLINE inline double skip_score(const ProbView& v, const SkipProb& sp, int64_t in_s, int64_t in_e, const int* c,
                             bool* undefined) {
  const int E = v.E;
  int last = -1;
  for (int e = 0; e < E; ++e)
    if (c[e] >= 0 && (last < 0 || v.oe[e][c[e]] > v.oe[last][c[last]])) last = e;
  if (last < 0) { *undefined = true; return 0.0; }         // AllSkip2: the reference fails to unpack `return 0`
  double total = 0.0;
  int num = 0;
  for (int e = 0; e < E; ++e) {
    if (c[e] < 0) continue;
    const int64_t cs = v.os[e][c[e]], ce = v.oe[e][c[e]];
    const int8_t* po = sp.pred_order + e * TW_MAX_E;
    for (int q = 0; q < TW_MAX_E && po[q] >= 0; ++q) {
      const int b = po[q];
      if (!edge_primary(v, b, e)) continue;
      if (c[b] < 0) {
        if (v.pred[b] == 0) {                                 // FindValidAncestor -> None
          total = dadd(total, pair_cost(sp, E, 0, 1 + e, cs - in_s, undefined));
        } else {
          const int8_t* pb = sp.pred_order + b * TW_MAX_E;
          int la = -1;
          for (int r = 0; r < TW_MAX_E && pb[r] >= 0; ++r) {
            const int a = pb[r];
            if (c[a] >= 0 && (la < 0 || v.oe[a][c[a]] > v.oe[la][c[la]])) la = a;
          }
          if (la < 0) { *undefined = true; return 0.0; }     // a chain of skipped ancestors
          total = dadd(total, pair_cost(sp, E, 1 + la, 1 + e, cs - v.os[la][c[la]], undefined));   // (sic) its START
        }
        ++num;
        continue;
      }
      total = dadd(total, pair_cost(sp, E, 1 + b, 1 + e, cs - v.oe[b][c[b]], undefined));
      ++num;
    }
    if (v.pred[e] == 0) { total = dadd(total, pair_cost(sp, E, 0, 1 + e, cs - in_s, undefined)); ++num; }
    if (e == last) { total = dadd(total, pair_cost(sp, E, 1 + e, 0, in_e - ce, undefined)); ++num; }
  }
  return sp.normalized ? ddiv(total, (double)num) : total;
}

// A GIVEN tuple of in-span i (tw_skip_score_assignments), the skip regime's assess_in_span: `assign` is
// the batch's tw_pass_out.assign array in sorted-list indices (-1 NA, <= -2 a skip span, whichever);
// tks / tki (NULL: no margin) are the in-span's row of its top2 list holding tk_cnt entries.  The
// feasibility checks are the candidate filter and the DAG check skip_topk applies while it builds a
// tuple, the score is skip_score's, so a listed tuple gets its listed score bit for bit.
TW_HD_NOINLINE inline Assessment skip_assess_in_span(const ProbView& v, const SkipProb& sp, int i, const int32_t* assign,
                                     const double* tks, const int32_t* tki, int tk_cnt) {
  Assessment a{NAN, NAN, TW_ASSESS_SCORED};
  int c[TW_MAX_E];
  bool na = false, range = false;
  for (int e = 0; e < v.E; ++e) {
    c[e] = assign[v.tuple_off + (int64_t)e * v.n_in + i];
    if (c[e] == -1) na = true;
    else if (c[e] >= v.n_out[e]) range = true;
  }
  if (na || range) {
    a.code = na ? TW_ASSESS_NA : TW_ASSESS_RANGE;
    return a;
  }
  const int64_t in_s = v.is[i], in_e = v.ie[i];
  for (int e = 0; e < v.E; ++e)                                      // V3:328-333
    if (c[e] >= 0 && (v.os[e][c[e]] < in_s || v.oe[e][c[e]] > in_e)) {
      a.code = TW_ASSESS_CONTAIN;
      return a;
    }
  for (int e = 0; e < v.E; ++e)                                      // V3:335-347, as skip_topk
    for (int b = 0; b < e; ++b)
      if (c[e] >= 0 && (v.pred[e] >> b & 1u) && c[b] >= 0 && v.oe[b][c[b]] > v.os[e][c[e]]) {
        a.code = TW_ASSESS_ORDER;
        return a;
      }
  bool undefined = false;
  const double score = skip_score(v, sp, in_s, in_e, c, &undefined);
  if (undefined) {
    a.code = TW_SKIP_ASSESS_UNDEFINED;
    return a;
  }
  a.score = score;
  if (tks && tk_cnt > 0) {
    bool top = true;                                                 // skips at one position are one span here
    for (int e = 0; e < v.E; ++e) top = top && (tki[e] == c[e] || (tki[e] < -1 && c[e] < -1));
    a.margin = !top ? dsub(a.score, tks[0]) : tk_cnt > 1 ? dsub(tks[0], tks[1]) : INFINITY;
  }
  return a;
}

// FetchSkipFromWindow, V3:820-842: the least-used skip span of the in-span's time window, first on ties
// = round robin over the window's skip spans.  Returns the code -2 - g, or 0 for "none available".
TW_HD_NOINLINE inline int fetch_skip(const SkipProb& sp, int e, int w) {
  const int cnt = sp.skip_count[e * sp.n_win + w];
  if (cnt <= 0) return 0;
  const int f = sp.fetches[e * sp.n_win + w]++;
  return -2 - (sp.skip_base[e * sp.n_win + w] + f % cnt);
}

// One FindTopKAssignments call (V3:180-465) in the skip regime.  deleted: search the lists with the
// taken spans removed, in the CALLER's order (the copies V3:1104-1105 takes before TallySkipSpans sorts).
TW_HD_NOINLINE inline int skip_topk(const ProbView& v, const SkipProb& sp, SkipShared& sh, int i, int w, bool deleted,
                         const uint32_t* taken, const int64_t* taken_off, int* err_flag) {
  const int E = v.E;
  const int64_t in_s = v.is[i], in_e = v.ie[i];
  for (int e = 0; e < E; ++e) {
    int nc = 0;
    for (int x = lower_bound(v.os[e], v.n_out[e], in_s); x < v.n_out[e] && v.os[e][x] <= in_e; ++x) {
      if (v.oe[e][x] > in_e) continue;
      if (deleted) {
        const int64_t bit = taken_off[e] + x;
        if (taken[bit >> 5] >> (bit & 31) & 1u) continue;
      }
      if (nc == kSkipCand) { raise(err_flag, TW_ERR_RANGE_LIMIT); return 0; }
      // insertion by position in the caller's list (identity when the caller's list is sorted)
      int pos = nc;
      if (deleted) {
        const int key = sp.entry_pos[e][x];
        while (pos > 0 && sp.entry_pos[e][sh.cand[e][pos - 1]] > key) { sh.cand[e][pos] = sh.cand[e][pos - 1]; --pos; }
      }
      sh.cand[e][pos] = x;
      ++nc;
    }
    sh.ncand[e] = nc;
  }
  TopK& tk = sh.tk;
  tk.clear();
  int leaves = 0;
  int c[TW_MAX_E], pos[TW_MAX_E];
  int e = 0;
  pos[0] = 0;
  while (e >= 0) {
    bool have = false;
    if (pos[e] < sh.ncand[e]) {
      const int x = sh.cand[e][pos[e]++];
      const int64_t s = v.os[e][x];
      bool ok = true;
      for (int b = 0; b < e && ok; ++b)
        if ((v.pred[e] >> b & 1u) && c[b] >= 0 && v.oe[b][c[b]] > s) ok = false;    // V3:335-347
      if (!ok) continue;
      c[e] = x;
      have = true;
    } else if (pos[e] == sh.ncand[e]) {
      ++pos[e];
      const int code = fetch_skip(sp, e, w);                  // the None sentinel, V3:231-234, :316-320
      if (code == 0) continue;
      c[e] = code;
      have = true;
    } else {
      --e;
      continue;
    }
    if (!have) continue;
    if (e < E - 1) { ++e; pos[e] = 0; continue; }
    // ---- leaf
    ++leaves;
    bool undefined = false;
    const double score = skip_score(v, sp, in_s, in_e, c, &undefined);
    if (undefined) { raise(err_flag, TW_ERR_REFERENCE_UNDEFINED); return leaves; }
    for (int h = 0; h < tk.n; ++h) {           // equal scores: heapq would compare a skip span with a real one
      const int slot = tk.heap[h];
      if (tk.score[slot] == score)
        for (int q = 0; q < E; ++q)
          if (tk.idx[slot][q] != c[q]) {
            if (tk.idx[slot][q] < 0 || c[q] < 0) { raise(err_flag, TW_ERR_REFERENCE_UNDEFINED); return leaves; }
            break;
          }
    }
    topk_offer(v, tk, score, c);
  }
  topk_finish(v, tk);
  return leaves;
}

// Exact MWIS of a window with weights added exactly (see oracle/tw_oracle_skip.py: exact_mwis): per
// connected component, depth-first over "rank r or none", first optimum wins.
TW_HD_NOINLINE inline long long skip_mwis(SkipShared& sh, int E, int nw, long long node_limit) {
  WindowBuf& wb = sh.wb;
  for (int k = 0; k < nw; ++k) { wb.adj[k] = window_adjacency(wb, E, nw, k); wb.chosen[k] = -1; }
  long long nodes = 0;
  uint32_t todo = nw >= 32 ? 0xffffffffu : ((1u << nw) - 1u);
  while (todo) {
    int seed = lowest_bit(todo);
    uint32_t comp = 1u << seed, frontier = comp;
    while (frontier) {
      const int k = lowest_bit(frontier);
      frontier &= frontier - 1u;
      const uint32_t nb = wb.adj[k] & ~comp;
      comp |= nb;
      frontier |= nb;
    }
    todo &= ~comp;
    int* member = sh.win_member;
    int m = 0;
    for (int k = 0; k < nw; ++k)
      if (comp >> k & 1u) member[m++] = k;
    long long wq[TW_WINDOW_CAP][TW_K];
    long long ub[TW_WINDOW_CAP + 1];
    ub[m] = 0;
    for (int l = m - 1; l >= 0; --l) {
      const int k = member[l];
      long long mx = 0;
      for (int r = 0; r < wb.cnt[k]; ++r) {
        wq[l][r] = (long long)((TW_WEIGHT_OFFSET + wb.score[k][r]) * kFixedScale);
        mx = wq[l][r] > mx ? wq[l][r] : mx;
      }
      ub[l] = ub[l + 1] + mx;
    }
    int choice[TW_WINDOW_CAP], best[TW_WINDOW_CAP], iter[TW_WINDOW_CAP + 1];
    long long cur[TW_WINDOW_CAP + 1];
    long long best_w = -1;
    for (int l = 0; l < m; ++l) best[l] = -1;
    int level = 0;
    cur[0] = 0;
    iter[0] = 0;
    while (level >= 0) {
      if (level == m) {
        ++nodes;
        if (cur[m] > best_w) {
          best_w = cur[m];
          for (int l = 0; l < m; ++l) best[l] = choice[l];
        }
        --level;
        continue;
      }
      const int k = member[level];
      if (iter[level] == 0) {
        ++nodes;
        if (nodes > node_limit) return -1;
        if (cur[level] + ub[level] <= best_w) { --level; continue; }
      }
      const int r = iter[level]++;
      if (r > wb.cnt[k]) { --level; continue; }
      if (r == wb.cnt[k]) {
        choice[level] = -1;
        cur[level + 1] = cur[level];
        ++level;
        iter[level] = 0;
        continue;
      }
      if (!(wq[level][r] > 0)) continue;
      bool ok = true;
      for (int l = 0; l < level && ok; ++l)
        if (choice[l] >= 0 && tuples_conflict(wb.idx[k][r], wb.idx[member[l]][choice[l]], E)) ok = false;
      if (!ok) continue;
      choice[level] = r;
      cur[level + 1] = cur[level] + wq[level][r];
      ++level;
      iter[level] = 0;
    }
    for (int l = 0; l < m; ++l) wb.chosen[member[l]] = best[l];
  }
  return nodes;
}

// ---------------------------------------------------------------------------------------------
// Candidate sets of CreateWindows2 on the caller's (possibly unsorted) lists -> PerfectCut flags.
// Sets are bitmaps over the caller's positions; three rotate: the in-span's, the previous in-span's,
// and the one of prev_index (V3:1026-1032).
// ---------------------------------------------------------------------------------------------
struct EntryList {
  const int64_t* s;
  const int64_t* e;
  const int32_t* of_entry;
  int n;
  TW_HD int64_t start(int x) const { return s[of_entry[x]]; }
  TW_HD int64_t end(int x) const { return e[of_entry[x]]; }
};
TW_HD_NOINLINE inline int entry_bisect_left(const EntryList& l, int64_t key) {
  int lo = 0, hi = l.n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (l.start(mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}
TW_HD_NOINLINE inline int entry_bisect_right(const EntryList& l, int64_t key) {
  int lo = 0, hi = l.n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (key < l.start(mid)) hi = mid; else lo = mid + 1;
  }
  return lo;
}

TW_HD_NOINLINE inline void set_clear(uint32_t* w, int words, SkipShared& sh, int slot) {
  if (sh.ntouched[slot] > kSkipTouched) {
    for (int q = 0; q < words; ++q) w[q] = 0u;
  } else {
    for (int q = 0; q < sh.ntouched[slot]; ++q) w[sh.touched[slot][q]] = 0u;
  }
  sh.ntouched[slot] = 0;
}
TW_HD_NOINLINE inline void set_add(uint32_t* w, SkipShared& sh, int slot, int bit) {
  const int q = bit >> 5;
  if (w[q] == 0u) {
    if (sh.ntouched[slot] < kSkipTouched) sh.touched[slot][sh.ntouched[slot]] = q;
    ++sh.ntouched[slot];                      // beyond kSkipTouched: cleared wholesale
  }
  w[q] |= 1u << (bit & 31);
}
TW_HD_NOINLINE inline bool sets_disjoint(const uint32_t* a, const uint32_t* b, int words, const SkipShared& sh, int slot_a) {
  if (sh.ntouched[slot_a] > kSkipTouched) {
    for (int q = 0; q < words; ++q)
      if (a[q] & b[q]) return false;
    return true;
  }
  for (int t = 0; t < sh.ntouched[slot_a]; ++t) {
    const int q = sh.touched[slot_a][t];
    if (a[q] & b[q]) return false;
  }
  return true;
}

TW_HD_NOINLINE inline void literal_candidates(const ProbView& v, const EntryList* el, const int* set_off, int i, uint32_t* w,
                                   SkipShared& sh, int slot) {
  const int E = v.E;
  const int64_t in_s = v.is[i], in_e = v.ie[i];
  int lo[TW_MAX_E], hi[TW_MAX_E];
  for (int e = 0; e < E; ++e) { lo[e] = el[e].n - 1; hi[e] = 0; }
  for (int node = E - 1; node >= 0; --node) {               // reverse topological order, V3:191-215
    int64_t exit_t = in_e;
    for (int nb = node + 1; nb < E; ++nb)
      if (v.pred[nb] >> node & 1u) {
        int idx = hi[nb];
        if (idx < 0) idx += el[nb].n;                        // Python's negative index
        const int64_t t = el[nb].start(idx);
        exit_t = t < exit_t ? t : exit_t;
      }
    lo[node] = entry_bisect_left(el[node], in_s);
    hi[node] = entry_bisect_right(el[node], exit_t) - 1;
  }
  int x[TW_MAX_E], c[TW_MAX_E];
  int e = 0;
  x[0] = lo[0];
  while (e >= 0) {
    if (x[e] > hi[e] || x[e] >= el[e].n) { --e; continue; }
    const int xi = x[e]++;
    const int64_t s = el[e].start(xi), en = el[e].end(xi);
    if (in_s > s || en > in_e) continue;
    bool ok = true;
    for (int b = 0; b < e && ok; ++b)
      if ((v.pred[e] >> b & 1u) && el[b].end(c[b]) > s) ok = false;
    if (!ok) continue;
    c[e] = xi;
    if (e == E - 1) {
      for (int q = 0; q < E; ++q) set_add(w, sh, slot, set_off[q] + c[q]);
      continue;
    }
    ++e;
    x[e] = lo[e] < 0 ? 0 : lo[e];
  }
}

// One service through the whole skip-regime iteration.  `sh`: work buffers (shared memory in the kernel).
// Returns TW_OK or the status the caller reports.
TW_HD_NOINLINE inline int skip_solve_problem(const tw_batch& b, int p, const tw_skip_desc& sd, const tw_skip_out& out,
                                             uint32_t* taken, uint32_t* set_scratch, const int64_t* prob_set_off,
                                             int32_t* win_scratch, long long node_limit, SkipShared& sh) {
  int status = TW_OK;
  int* err_flag = &status;
  ProbView v;
  if (load_view(b, p, v) != TW_OK) return TW_ERR_INVALID;
  const int E = v.E, n = v.n_in;
  SkipProb sp = skip_prob(sd, v, p);
  sp.skip_base = win_scratch + 2 * sd.prob_cnt_off[p];
  sp.fetches = sp.skip_base + (size_t)E * sp.n_win;
  EntryList el[TW_MAX_E];
  int set_off[TW_MAX_E];
  int64_t taken_off[TW_MAX_E];
  int set_bits = 0;
  for (int e = 0; e < E; ++e) {
    el[e].s = v.os[e]; el[e].e = v.oe[e]; el[e].of_entry = sp.sorted_of_entry[e]; el[e].n = v.n_out[e];
    set_off[e] = set_bits;
    set_bits += (v.n_out[e] + 31) & ~31;
    taken_off[e] = v.out_off[e] + 32 * (int64_t)(v.ep0 + e);   // word-aligned per ep (as the stitch kernel)
    int run = 0;
    for (int w = 0; w < sp.n_win; ++w) {
      sp.skip_base[e * sp.n_win + w] = run;
      const int cnt = sp.skip_count[e * sp.n_win + w];
      run += cnt > 0 ? cnt : 0;
      sp.fetches[e * sp.n_win + w] = 0;
    }
  }
  // taken bits of this problem start clear
  for (int e = 0; e < E; ++e)
    for (int64_t q = taken_off[e] >> 5; q <= (taken_off[e] + v.n_out[e]) >> 5; ++q) taken[q] = 0u;

  // ---- 1. PerfectCut flags (V3:1024-1039) from the literal candidate sets
  const int words = set_bits >> 5;
  uint32_t* sets = set_scratch + 3 * prob_set_off[p];
  uint32_t* buf[3] = {sets, sets + words, sets + 2 * (size_t)words};
  for (int q = 0; q < 3 * words; ++q) sets[q] = 0u;
  sh.ntouched[0] = sh.ntouched[1] = sh.ntouched[2] = 0;
  uint8_t* cut = out.cut + v.in_off;
  int s_cur = 0, s_last = 1;                  // buffer slots of set(i) and set(i-1); slot 2 = set(prev_index)
  const int s_prev = 2;
  int prev_index = 0;
  for (int i = 0; i < n; ++i) {
    cut[i] = 0;
    const bool inner = i >= 1 && i <= n - 2;
    if (inner && (i == 1 || v.ie[i - 1] >= v.ie[prev_index])) {      // V3:1026-1032
      prev_index = i - 1;
      set_clear(buf[s_prev], words, sh, s_prev);
      if (sh.ntouched[s_last] > kSkipTouched) {
        for (int q = 0; q < words; ++q) buf[s_prev][q] = buf[s_last][q];
      } else {
        for (int t = 0; t < sh.ntouched[s_last]; ++t) {
          const int q = sh.touched[s_last][t];
          buf[s_prev][q] = buf[s_last][q];
          sh.touched[s_prev][t] = q;
        }
      }
      sh.ntouched[s_prev] = sh.ntouched[s_last];
    }
    set_clear(buf[s_cur], words, sh, s_cur);
    literal_candidates(v, el, set_off, i, buf[s_cur], sh, s_cur);
    if (inner) {
      const bool disjoint = sets_disjoint(buf[s_cur], buf[s_prev], words, sh, s_cur);
      cut[i] = (uint8_t)(disjoint && v.ie[prev_index] <= v.ie[i]);
    }
    const int t = s_cur; s_cur = s_last; s_last = t;
  }

  // ---- 2. the hot loop, one iteration (V3:1159-1219)
  WindowCursor wc;
  wc.init();
  int nw = 0, w_first = 0;
  int not_best = 0, unassigned = 0;
  long long max_nodes = 0;
  const bool want_topk = out.pass.topk_score != nullptr;
  for (int i = 0; i < n; ++i) {
    // time window of the in-span (FindWindow, V3:827-831): the last start <= key, first of equal starts
    int w = upper_bound(sp.win_start, sp.n_win, v.is[i]) - 1;
    if (w < 0) return TW_ERR_REFERENCE_UNDEFINED;
    while (w > 0 && sp.win_start[w - 1] == sp.win_start[w]) --w;
    const int64_t gi = v.in_off + i;
    // top_k on the lists with deletion (V3:1182)
    const int leaves = skip_topk(v, sp, sh, i, w, true, taken, taken_off, err_flag);
    if (status != TW_OK) return status;
    out.pass.n_cand[gi] = leaves;
    if (nw == 0) w_first = i;
    sh.wb.cnt[nw] = sh.tk.n;
    for (int r = 0; r < sh.tk.n; ++r) {
      sh.wb.score[nw][r] = sh.tk.score[r];
      for (int e = 0; e < E; ++e) sh.wb.idx[nw][r][e] = sh.tk.idx[r][e];
    }
    if (want_topk)
      store_topk_row(sh.tk, E, out.pass.topk_score + gi * TW_K,
                     out.pass.topk_idx + TW_K * (v.tuple_off + (int64_t)i * E), out.pass.topk_cnt + gi);
    ++nw;
    // top_k_2 on the undeleted, sorted lists (V3:1185) -> all_topk_assignments
    skip_topk(v, sp, sh, i, w, false, taken, taken_off, err_flag);
    if (status != TW_OK) return status;
    store_topk_row(sh.tk, E, out.top2_score + gi * TW_K, out.top2_idx + TW_K * (v.tuple_off + (int64_t)i * E),
                   out.top2_cnt + gi);
    if (!wc.ends_at(i, n, cut)) continue;
    // ---- window end: MWIS, assignment, deletion
    const long long nodes = skip_mwis(sh, E, nw, node_limit);
    if (nodes < 0) return TW_ERR_MWIS_LIMIT;
    max_nodes = nodes > max_nodes ? nodes : max_nodes;
    for (int k = 0; k < nw; ++k) {
      const int ii = w_first + k;
      const int r = sh.wb.chosen[k];
      out.pass.mis_rank[v.in_off + ii] = (int8_t)r;
      if (r < 0) { ++unassigned; ++not_best; }
      else if (r != 0) ++not_best;
      for (int e = 0; e < E; ++e) {
        int a = -1;
        if (r >= 0) {
          const int c = sh.wb.idx[k][r][e];
          if (c >= 0) {
            a = c;
            const int64_t bit = taken_off[e] + c;
            taken[bit >> 5] |= 1u << (bit & 31);
          } else {
            a = -2;                                        // ('Skip', 'Skip'), V1:449-451
          }
        }
        out.pass.assign[v.tuple_off + (int64_t)e * n + ii] = a;
      }
    }
    nw = 0;
  }
  int32_t* ctr = out.pass.counters + 4 * p;
  ctr[0] = not_best;
  ctr[1] = unassigned;
  ctr[2] = (int32_t)(max_nodes > 0x7fffffff ? 0x7fffffff : max_nodes);
  ctr[3] = 0;
  return status;
}

}  // namespace tw
