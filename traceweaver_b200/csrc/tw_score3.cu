// tw_score3.cu — candidate enumeration + likelihood scoring + top-K on the undeleted lists.
//
// Replaces (reference: .../algorithms/traceweaver_v3.py = V3, traceweaver_v1.py = V1)
//   FindTopKAssignments(K=5, out_span_partitions)   V3:1185  (DfsTraverseX V3:292-351,
//       ScoreAssignmentAsPerInvocationGraph V1:259-361, GetEpPairCost V1:117-139)
//   the enumeration half of CreateWindows2            V3:1041-1051 (candidate maps; the PerfectCut
//       flags are derived from the maps by k_cut below, V3:1024-1039)
//
// Mapping to the machine.  HBM-bound integer / f64 work, no tensor cores.  The workload is heavy
// tailed: the median in-span has ONE feasible tuple, the mean ~10 candidate combinations, the
// tail thousands.  So nothing after the range search is indexed by in-span:
//
//   * one CTA = one TILE of 128 consecutive in-spans of one service, one warp = 32 of them.  Both
//     sides are sorted by start, so the tile's candidates are one contiguous slice of each ep's
//     list; the slice bounds come from a pre-pass (k_tile_meta, once per bound batch) and the
//     slices are brought into shared memory with 1-D bulk copies (cp.async.bulk -> UBLKCP)
//     completing on an mbarrier.  After that barrier the four warps never synchronise again.
//   * per warp, all per-in-span state lives in REGISTERS as packed words (candidate counts 8 bits
//     per ep, range offsets 16 bits per ep, tuples 6 bits per ep): the kernel is templated on E
//     and has no local-memory arrays (0 bytes of stack).
//   * work items are flattened over the warp's 32 in-spans with prefix sums and handed out
//     lane-strided; the owner of an item is found by a 5-step binary search of the prefix over
//     shuffles:
//       1a  slots   every likelihood term value any tuple can use (r_e values per root / last
//                   term, r_b * r_e per edge term): decode, validity, dt -> compacted list
//       1b  values  the FP64 work (GetEpPairCost): every lane evaluates one VALID slot
//       2a  combos  every element of every in-span's candidate product space: containment and
//                   DAG-order tests -> compacted list of feasible tuples (+ candidate maps)
//       2b  scores  every lane sums one feasible tuple's table entries (reference term order)
//       2c  top-K   the owner lane walks its (contiguous) segment of the list; 5 keys in
//                   registers, compare-exchange insertion, no atomics
//   * results leave through shared memory as coalesced 128-bit stores.
//
// Anything this kernel cannot do EXACTLY is not approximated: the tile is flagged and redone by
// the sequential kernel (k_score<32,64>, tw_score.cu): more than 64 candidates of one ep in an
// in-span's range, more than 2^24 combinations, a slice that does not fit the staging buffer, two
// tuples of one in-span with the same score (the reference's heap order decides), a NaN score.
#include "tw_kernels.cuh"

namespace tw {

// optional phase timers / work counters (build with -DTW_PROFILE_PHASES; scripts/score_phase_profile.py)
#ifdef TW_PROFILE_PHASES
__device__ unsigned long long g_score_phase[24];
#define TW_CPHASE(k)                                                                 \
  do {                                                                               \
    if (lane == 0) {                                                                 \
      long long _now = clock64();                                                    \
      atomicAdd(&g_score_phase[k], (unsigned long long)(_now - _cp_t0));             \
      _cp_t0 = _now;                                                                 \
    }                                                                                \
  } while (0)
#define TW_CCOUNT(k, v) do { if (lane == 0) atomicAdd(&g_score_phase[k], (unsigned long long)(v)); } while (0)
extern "C" int tw_debug_score_phases(unsigned long long* out24, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out24, g_score_phase, sizeof(unsigned long long) * 24);
  if (e != cudaSuccess) return -2;
  if (reset) {
    unsigned long long z[24] = {0};
    cudaMemcpyToSymbol(g_score_phase, z, sizeof z);
  }
  return 0;
}
#else
#define TW_CPHASE(k) do { } while (0)
#define TW_CCOUNT(k, v) do { } while (0)
#endif

#ifndef TW_S3_TBL
#define TW_S3_TBL 416          // term-table slots per warp per round
#define TW_S3_ENT 192          // feasible tuples per warp between two flushes of the list
#define TW_S3_PRM_TERMS 16     // likelihood records staged in shared memory (else read in place)
#endif
constexpr int kS3Tbl = TW_S3_TBL;
constexpr int kS3Ent = TW_S3_ENT;
constexpr int kS3Prm = TW_S3_PRM_TERMS * TW_MIX_REC;
constexpr int kS3Warps = kS3Threads / 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kS3MaxR = 64;                 // candidates of one ep in one in-span's range
constexpr int kS3RankMax = 12;              // segments up to this many feasible tuples are ranked entry-parallel
constexpr long long kS3MaxP = 1LL << 24;    // combinations of one in-span

// ---- PTX: mbarrier + 1-D bulk copy (TMA engine, SASS UBLKCP) ---------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LAB_DONE;\n"
      "bra LAB_WAIT;\n"
      "LAB_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

// ---- packed per-in-span state -------------------------------------------------------------------
// rp : candidate count of ep e in bits [8e, 8e+8)     (<= 64)
// lp : offset of the first candidate of ep e inside the staged slice, bits [16e, 16e+16)
// xp : a tuple, candidate offset of ep e in bits [6(E-1-e), +6): numeric order == DFS leaf order
template <int E>
struct S3Pack {
  static constexpr bool kWide = E > 4;
  using rp_t = typename std::conditional<kWide, unsigned long long, uint32_t>::type;
  using xp_t = typename std::conditional<kWide, unsigned long long, uint32_t>::type;
  static constexpr int kLW = (E + 3) / 4;   // 64-bit words of lp
};

template <int E>
struct S3Lo { unsigned long long w[S3Pack<E>::kLW]; };

template <int E>
__device__ __forceinline__ int lo_get(const S3Lo<E>& l, int e) {
  unsigned long long w = l.w[0];
  if (S3Pack<E>::kLW > 1 && e >= 4) w = l.w[S3Pack<E>::kLW - 1];
  return (int)((w >> ((e & 3) * 16)) & 0xffffull);
}
template <int E>
__device__ __forceinline__ S3Lo<E> lo_shfl(const S3Lo<E>& l, int src) {
  S3Lo<E> o;
#pragma unroll
  for (int q = 0; q < S3Pack<E>::kLW; ++q) o.w[q] = __shfl_sync(kFull, l.w[q], src);
  return o;
}
template <class RP>
__device__ __forceinline__ int r_get(RP rp, int e) { return (int)((rp >> (8 * e)) & 0xff); }

// floor(idx / r) for idx < 2^24, 1 <= r <= 64: one multiply by ceil(2^32 / r)
__device__ __forceinline__ unsigned div_small(unsigned idx, int r, const uint32_t* __restrict__ magic) {
  return r == 1 ? idx : __umulhi(idx, magic[r]);
}

// ---- shared memory ---------------------------------------------------------------------------------
template <int E>
struct S3Warp {
  alignas(16) double tbl[kS3Tbl];             // term tables of the round; output staging afterwards
  unsigned long long ent_key[kS3Ent];         // order-preserving score keys of the feasible tuples
  typename S3Pack<E>::xp_t ent_xp[kS3Ent];
  int64_t ins[32], ine[32];
  alignas(16) uint32_t used[32][E][kNarrowW]; // candidate maps (V3:1043-1051)
  int seg_lo[32], seg_hi[32];
  uint16_t val_slot[kS3Tbl];                  // compacted valid slots of the current term: slot | batch << 12
  unsigned long long top_key[32][TW_K];       // quick ranking (2c): rank r of in-span j
  typename S3Pack<E>::xp_t top_xp[32][TW_K];
  uint8_t ent_j[kS3Ent];
  uint8_t seg_quick[32];
};

template <int E>
struct S3Smem {
  static constexpr int kStage = E <= 4 ? 704 : 1536;   // staged out spans per tile, all eps
  alignas(16) int64_t st_s[kStage];
  alignas(16) int64_t st_e[kStage];
  alignas(8) uint64_t bar;
  double prm[kS3Prm];
  double etab[64];
  S3Warp<E> w[kS3Warps];
  uint32_t magic[kS3MaxR + 1];
  int woff_s[E], woff_e[E], win_a[E], win_n[E];
  uint32_t pred[E];
  int8_t tsrc[TW_MAX_TERMS];
  uint8_t tep[TW_MAX_TERMS];
};

__device__ __forceinline__ double key_to_score3(unsigned long long k) {
  unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffULL) : ~k;
  return __longlong_as_double((long long)u);
}

// one likelihood value on a rare path (kept out of line so the hot loops stay small)
__device__ __noinline__ double term_logpdf_cold(int mode, const double* rec_base, int n_terms, int brel, int t,
                                                const double* etab, double dt) {
  ParamView pv;
  pv.mode = mode;
  pv.gauss = rec_base + brel * n_terms * TW_GAUSS_REC;
  pv.mix = rec_base;
  pv.etab = etab;
  return term_logpdf(pv, t, dt);
}

// coalesced copy of `nwords` 32-bit words from shared to global memory by one warp: 128-bit stores
// when the destination is 16-byte aligned (it is, for the layouts the host mirror builds)
__device__ __forceinline__ void warp_copy_out(void* dst, const void* src, int nwords, int lane) {
  if (((((uintptr_t)dst) | ((uintptr_t)src)) & 15u) == 0) {
    const int n4 = nwords >> 2;
    const int4* s4 = reinterpret_cast<const int4*>(src);
    int4* d4 = reinterpret_cast<int4*>(dst);
    for (int k = lane; k < n4; k += 32) d4[k] = s4[k];
    const int* s1 = reinterpret_cast<const int*>(src);
    int* d1 = reinterpret_cast<int*>(dst);
    for (int k = (n4 << 2) + lane; k < nwords; k += 32) d1[k] = s1[k];
  } else {
    const int* s1 = reinterpret_cast<const int*>(src);
    int* d1 = reinterpret_cast<int*>(dst);
    for (int k = lane; k < nwords; k += 32) d1[k] = s1[k];
  }
}

// first lane whose inclusive prefix exceeds `item` (prefix is non-decreasing over the lanes)
__device__ __forceinline__ int owner_of(int incl, int item) {
  int j = 0;
#pragma unroll
  for (int step = 16; step > 0; step >>= 1) {
    const int v = __shfl_sync(kFull, incl, j + step - 1);
    if (v <= item) j += step;
  }
  return j;
}

template <int E>
__global__ void __launch_bounds__(kS3Threads, E <= 4 ? 4 : 2)
k_score3(tw_batch b, tw_params prm, int has_params, int keep_windows, tw_score_out out, TileList tiles,
         const int32_t* __restrict__ tile_win, uint8_t* __restrict__ overflow_flag) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  S3Smem<E>& sm = *reinterpret_cast<S3Smem<E>*>(smem_raw);
  using RP = typename S3Pack<E>::rp_t;
  using XP = typename S3Pack<E>::xp_t;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int t = blockIdx.x;
#ifdef TW_PROFILE_PHASES
  long long _cp_t0 = clock64();
#endif
  if (keep_windows && overflow_flag[t]) return;      // the sequential kernel owns this tile
  const int p = tiles.tile_prob[t];
  const int i0 = tiles.tile_start[t];
  const int32_t* tw = tile_win + (size_t)t * 2 * TW_MAX_E;

  // ---- problem header (uniform loads)
  const int ep0 = b.prob_ep_off[p];
  const int64_t in_off = b.prob_in_off[p];
  const int n = (int)(b.prob_in_off[p + 1] - in_off);
  const int64_t tuple_off = b.prob_tuple_off[p];
  const int term0 = b.ep_term_off[ep0];
  const int n_terms = b.ep_term_off[ep0 + E] - term0;
  const int cnt = min(kS3Tile, n - i0);

  // ---- staging layout (every thread, from the tile's slice bounds): ep e occupies an even number
  // of elements; a slice whose global address is 8 mod 16 starts at an odd element so the bulk
  // copy (16-byte granules) is aligned on both sides
  int tot = 0;
#pragma unroll
  for (int e = 0; e < E; ++e) tot += (tw[2 * e + 1] + 3) & ~1;
  if (tot > S3Smem<E>::kStage) {
    if (tid == 0 && !keep_windows) overflow_flag[t] = 1;
    if (tid == 0) { TW_CCOUNT(15, 1); }           // staging overflow
    return;
  }
  if (tid == 0) mbar_init(&sm.bar, 2 * E);
  __syncthreads();                                   // mbarrier initialised

  // ---- bulk copies: thread 2e stages the start times of ep e, thread 2e+1 the end times
  if (tid < 2 * E) {
    const int e = tid >> 1, which = tid & 1;
    int off = 0;
    for (int q = 0; q < e; ++q) off += (tw[2 * q + 1] + 3) & ~1;
    const int a = tw[2 * e], ne = tw[2 * e + 1];
    const int64_t* g = (which ? b.out_end : b.out_start) + b.ep_out_off[ep0 + e] + a;
    const int mis = (int)((((uintptr_t)g) >> 3) & 1u);
    int64_t* d = (which ? sm.st_e : sm.st_s) + off + mis;      // window element k lives at d[k]
    const int body = (ne - mis) > 0 ? ((ne - mis) & ~1) : 0;
    mbar_arrive_expect_tx(&sm.bar, (uint32_t)body * 8u);
    if (body > 0) bulk_g2s(d + mis, g + mis, (uint32_t)body * 8u, &sm.bar);
    if (mis && ne > 0) d[0] = g[0];                              // unaligned head
    if (ne - mis > body) d[ne - 1] = g[ne - 1];                  // odd tail
    if (which) sm.woff_e[e] = off + mis;
    else { sm.woff_s[e] = off + mis; sm.win_a[e] = a; sm.win_n[e] = ne; }
  }
  // ---- while the copies are in flight: tables, parameters, the own in-span
  if (tid < 64) sm.etab[tid] = c_exp2_64[tid];
  for (int r = tid; r <= kS3MaxR; r += kS3Threads) {
    sm.magic[r] = r >= 2 ? (uint32_t)(0xffffffffu / (uint32_t)r) + 1u : 0u;
  }
  if (tid < n_terms) {
    const int tg = term0 + tid;
    sm.tsrc[tid] = b.term_src[tg];
    int e = 0;
#pragma unroll
    for (int q = 1; q < E; ++q)
      if (tg >= b.ep_term_off[ep0 + q]) e = q;
    sm.tep[tid] = (uint8_t)e;
  }
  if (tid < E) sm.pred[tid] = b.ep_pred_mask[ep0 + tid];
  // likelihood parameters of the tile: staged when they fit, else read in place
  const int batch0 = i0 / TW_PARAM_BATCH;
  const double* prm_base = nullptr;
  if (has_params) {
    const double* src;
    int nrec;
    if (prm.mode == TW_PARAMS_GAUSS_BATCHED) {
      nrec = 3 * n_terms * TW_GAUSS_REC;          // a 128-span tile touches at most three 100-span batches
      const int nb = (n + TW_PARAM_BATCH - 1) / TW_PARAM_BATCH;
      src = prm.gauss + (prm.prob_gauss_off[p] + (int64_t)batch0 * n_terms) * TW_GAUSS_REC;
      const int avail = (nb - batch0) * n_terms * TW_GAUSS_REC;
      if (nrec > avail) nrec = avail;
    } else {
      src = prm.mix + (int64_t)term0 * TW_MIX_REC;
      nrec = n_terms * TW_MIX_REC;
    }
    prm_base = nrec <= kS3Prm ? sm.prm : src;
    if (nrec <= kS3Prm)
      for (int x = tid; x < nrec; x += kS3Threads) sm.prm[x] = src[x];
  }
  // own in-span
  const bool worker = tid < cnt;
  const int i = i0 + tid;
  int64_t in_s = 0, in_e = INT64_MIN;
  if (worker) { in_s = b.in_start[in_off + i]; in_e = b.in_end[in_off + i]; }
  S3Warp<E>& ws = sm.w[wid];
  ws.ins[lane] = in_s;
  ws.ine[lane] = in_e;
#pragma unroll
  for (int e = 0; e < E; ++e) { ws.used[lane][e][0] = 0u; ws.used[lane][e][1] = 0u; }
  mbar_wait(&sm.bar, 0);
  __syncthreads();                                   // heads / tails / layout visible

  TW_CPHASE(0);                                      // header, staging, barrier
  // ================= from here on the warps are independent =================
  const uint32_t* magic = sm.magic;
  // sink eps: the LAST term (V1:354-355) can only fall on an ep without DAG successors, unless end
  // times tie; those rare tuples evaluate the term on the spot
  uint32_t sink = (1u << E) - 1u;
#pragma unroll
  for (int e = 0; e < E; ++e) sink &= ~sm.pred[e];

  // ---- candidate ranges of the own in-span
  RP rp = 0;
  S3Lo<E> lp;
#pragma unroll
  for (int q = 0; q < S3Pack<E>::kLW; ++q) lp.w[q] = 0ull;
  bool anomaly = false;
  long long P = worker ? 1 : 0;
#pragma unroll
  for (int e = 0; e < E; ++e) {
    const int64_t* s = sm.st_s + sm.woff_s[e];
    const int ne = sm.win_n[e];
    int lo = 0, r = 0;
    if (worker) {
      lo = lower_bound(s, ne, in_s);
      while (lo + r < ne && s[lo + r] <= in_e && r <= kS3MaxR) ++r;
    }
    if (r > kS3MaxR) { anomaly = true; r = 0; }
    rp |= (RP)r << (8 * e);
    lp.w[e >> 2] |= (unsigned long long)lo << ((e & 3) * 16);
    P *= r;
  }
  if (P > kS3MaxP) { anomaly = true; P = 0; }
  if (__any_sync(kFull, anomaly)) {
    if (lane == 0 && !keep_windows) overflow_flag[t] = 1;
    TW_CCOUNT(16, 1);                                // range wider than 64 / too many combinations (per warp)
    return;   // (with keep_windows the flag is already set: same data, same decision)
  }
  // table size: root / sink-last terms r_e, edge terms r_b * r_e
  int tsize = 0;
  if (has_params) {
    for (int tt = 0; tt < n_terms; ++tt) {
      const int e = sm.tep[tt], src = sm.tsrc[tt];
      const int re = r_get(rp, e);
      tsize += src >= 0 ? r_get(rp, src) * re : (src == TW_TERM_ROOT || (sink >> e & 1u)) ? re : 0;
    }
    if (P == 0) tsize = 0;
  }
  const bool direct = tsize > kS3Tbl;        // tables do not fit: terms are evaluated per feasible tuple

  TW_CPHASE(1);                                      // candidate ranges, table sizes
  // top-K of the own in-span: keys descending, 0 = empty
  unsigned long long tk0 = 0, tk1 = 0, tk2 = 0, tk3 = 0, tk4 = 0;
  XP tx0 = 0, tx1 = 0, tx2 = 0, tx3 = 0, tx4 = 0;
  int nfeas = 0;
  bool redo = false;
  bool pending = worker && P > 0;

  while (__any_sync(kFull, pending)) {
    // ---- admit a prefix of the pending in-spans whose tables fit
    const int tneed = pending && !direct ? tsize : 0;
    int tend = tneed;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(kFull, tend, d);
      if (lane >= d) tend += o;
    }
    const bool admitted = pending && tend <= kS3Tbl;
    const int tstart = tend - tneed;
    const int total_t = __reduce_max_sync(kFull, admitted ? tend : 0);
    const int cneed = admitted ? (int)P : 0;
    int cend = cneed;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(kFull, cend, d);
      if (lane >= d) cend += o;
    }
    const int cstart = cend - cneed;
    const int total_c = __shfl_sync(kFull, cend, 31);

    TW_CPHASE(2);                                    // admission
    TW_CCOUNT(10, total_t);
    TW_CCOUNT(11, total_c);
    TW_CCOUNT(12, 1);
    // ---- 1. term tables, TERM-MAJOR: for one term at a time the slots of all admitted in-spans are
    // flattened over the warp, so the term, its eps, the candidate-count fields and (mixture pass)
    // the likelihood record and its component count are warp-uniform: no per-slot term search, no
    // divergence inside GetEpPairCost (V1:117-139), only live mixture components are evaluated.
    // Slots no feasible tuple can use (containment / order fails) are never evaluated or read.
    {
      int o_run = tstart;                       // own table of the current term starts here
      for (int tt = 0; tt < n_terms && total_t > 0; ++tt) {
        const int e = sm.tep[tt], src = sm.tsrc[tt];
        const bool tabled = src >= 0 || src == TW_TERM_ROOT || (sink >> e & 1u);
        const int re_own = r_get(rp, e);
        const int size = (admitted && !direct && tabled) ? (src >= 0 ? r_get(rp, src) * re_own : re_own) : 0;
        int incl = size;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int o = __shfl_up_sync(kFull, incl, d);
          if (lane >= d) incl += o;
        }
        const int total = __shfl_sync(kFull, incl, 31);
        const int excl = incl - size;
        const double* rec_mix = prm_base + tt * TW_MIX_REC;
        int nv = 0;
        for (int base = 0; base < total; base += 32) {
          const int s = base + lane;
          const bool act = s < total;
          const int j = owner_of(incl, act ? s : total - 1);
          const RP rpj = __shfl_sync(kFull, rp, j);
          const S3Lo<E> lpj = lo_shfl<E>(lp, j);
          const int l = s - __shfl_sync(kFull, excl, j);
          const int tb = __shfl_sync(kFull, o_run, j);
          const int re = r_get(rpj, e);
          const int64_t je = ws.ine[j];
          bool valid = act;
          double dt = 0.0;
          if (src >= 0) {
            const int xb = (int)div_small((unsigned)l, re, magic), xe = l - xb * re;
            const int64_t eb = sm.st_e[sm.woff_e[src] + lo_get<E>(lpj, src) + xb];
            const int pe = lo_get<E>(lpj, e) + xe;
            const int64_t sv = sm.st_s[sm.woff_s[e] + pe];
            valid = valid && eb <= je && sm.st_e[sm.woff_e[e] + pe] <= je && eb <= sv;
            dt = (double)(sv - eb);                                              // V1:345
          } else {
            const int pos = lo_get<E>(lpj, e) + l;
            const int64_t en = sm.st_e[sm.woff_e[e] + pos];
            valid = valid && en <= je;
            dt = src == TW_TERM_ROOT ? (double)(sm.st_s[sm.woff_s[e] + pos] - ws.ins[j])   // V1:349-350
                                     : (double)(je - en);                               // V1:354-355
          }
          // valid slots are compacted so that the FP64 work below runs on full warps
          const unsigned vm = __ballot_sync(kFull, valid);
          TW_CCOUNT(14, __popc(vm));
          if (valid) {
            const int pos = nv + __popc(vm & ((1u << lane) - 1u));
            const int brel = prm.mode == TW_PARAMS_GAUSS_BATCHED ? (i0 + wid * 32 + j) / TW_PARAM_BATCH - batch0 : 0;
            ws.tbl[tb + l] = dt;
            ws.val_slot[pos] = (uint16_t)((tb + l) | (brel << 12));
          }
          nv += __popc(vm);
        }
        __syncwarp();
        for (int vb = 0; vb < nv; vb += 32) {
          const int vi = vb + lane;
          if (vi < nv) {
            const int code = ws.val_slot[vi];
            const int slot = code & 0xfff;
            const double dt = ws.tbl[slot];
            double val;
            if (prm.mode == TW_PARAMS_GAUSS_BATCHED)
              val = gauss_logpdf(prm_base + ((code >> 12) * n_terms + tt) * TW_GAUSS_REC, dt);
            else
              val = mix_logpdf_tab_uniform(rec_mix, dt, sm.etab);
            ws.tbl[slot] = val;
          }
        }
        __syncwarp();
        o_run += size;
      }
    }
    __syncwarp();

    TW_CPHASE(3);                                    // term tables
    // ---- 2. combinations, in chunks of the entry list
    int n_ent = 0;
    int base = 0;
    while (true) {
      const int chunk_base = base;
      // 2a. feasibility (V3:328-347) -> compacted (tuple, owner) list, in DFS leaf order per owner
      for (; base < total_c && n_ent <= kS3Ent - 32; base += 32) {
        const int g = base + lane;
        const bool act = g < total_c;
        const int j = owner_of(cend, act ? g : total_c - 1);
        const RP rpj = __shfl_sync(kFull, rp, j);
        const S3Lo<E> lpj = lo_shfl<E>(lp, j);
        const int cstj = __shfl_sync(kFull, cstart, j);
        unsigned idx = act ? (unsigned)(g - cstj) : 0u;
        const int64_t je = ws.ine[j];
        int x[E];
        int64_t cs[E], ce[E];
        bool ok = act;
#pragma unroll
        for (int e = E - 1; e >= 0; --e) {
          if (e > 0) {
            const int re = r_get(rpj, e);
            const unsigned q = div_small(idx, re, magic);
            x[e] = (int)(idx - q * (unsigned)re);
            idx = q;
          } else {
            x[0] = (int)idx;
          }
        }
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int pos = lo_get<E>(lpj, e) + x[e];
          cs[e] = sm.st_s[sm.woff_s[e] + pos];
          ce[e] = sm.st_e[sm.woff_e[e] + pos];
          ok = ok && ce[e] <= je;
          const uint32_t pm = sm.pred[e];
#pragma unroll
          for (int bq = 0; bq < e; ++bq)
            if (pm >> bq & 1u) ok = ok && ce[bq] <= cs[e];
        }
        const unsigned m = __ballot_sync(kFull, ok);
        if (ok) {
          XP xp = 0;
#pragma unroll
          for (int e = 0; e < E; ++e) xp = (xp << 6) | (XP)x[e];
          const int pos = n_ent + __popc(m & ((1u << lane) - 1u));
          ws.ent_xp[pos] = xp;
          ws.ent_j[pos] = (uint8_t)j;
          if (!keep_windows) {
#pragma unroll
            for (int e = 0; e < E; ++e) atomicOr(&ws.used[j][e][x[e] >> 5], 1u << (x[e] & 31));
          }
        }
        n_ent += __popc(m);
      }
      __syncwarp();
      TW_CPHASE(4);                                  // 2a feasibility
      TW_CCOUNT(13, n_ent);
      // 2b. scores: sum of table entries in the reference's term order (V1:316-357)
      if (has_params) {
        for (int eb = 0; eb < n_ent; eb += 32) {
          const int en = eb + lane;
          const bool act = en < n_ent;
          const int j = act ? ws.ent_j[en] : 0;
          const XP xp = act ? ws.ent_xp[en] : (XP)0;
          const RP rpj = __shfl_sync(kFull, rp, j);
          const S3Lo<E> lpj = lo_shfl<E>(lp, j);
          const int tstj = __shfl_sync(kFull, tstart, j);
          const bool dirj = __shfl_sync(kFull, (int)direct, j) != 0;
          if (act) {
            int x[E];
            int64_t ce[E];
#pragma unroll
            for (int e = 0; e < E; ++e) {
              x[e] = (int)((xp >> (6 * (E - 1 - e))) & 63);
              ce[e] = sm.st_e[sm.woff_e[e] + lo_get<E>(lpj, e) + x[e]];
            }
            int last = 0;                       // max(..., key=end) keeps the first maximum (V1:314)
            int64_t last_end = ce[0];
#pragma unroll
            for (int e = 1; e < E; ++e)
              if (ce[e] > last_end) { last_end = ce[e]; last = e; }
            const int brel = prm.mode == TW_PARAMS_GAUSS_BATCHED ? (i0 + wid * 32 + j) / TW_PARAM_BATCH - batch0 : 0;
            double cost = 0.0;
            int o = tstj;
            for (int tt = 0; tt < n_terms; ++tt) {
              const int e = sm.tep[tt], src = sm.tsrc[tt];
              const int re = r_get(rpj, e);
              int xe = 0, xs = 0;
#pragma unroll
              for (int q = 0; q < E; ++q) {
                if (q == e) xe = x[q];
                if (q == src) xs = x[q];
              }
              const bool in_table = !dirj && (src != TW_TERM_LAST || (sink >> e & 1u));
              if (src == TW_TERM_LAST && e != last) {
                if (in_table) o += re;
                continue;
              }
              if (in_table) {
                cost = dadd(cost, ws.tbl[o + (src >= 0 ? xs * re : 0) + xe]);
                o += src >= 0 ? r_get(rpj, src) * re : re;
              } else {                          // tables too large, or a LAST term on a non-sink ep
                const int pe = lo_get<E>(lpj, e) + xe;
                int64_t d;
                if (src >= 0) d = sm.st_s[sm.woff_s[e] + pe] - sm.st_e[sm.woff_e[src] + lo_get<E>(lpj, src) + xs];
                else if (src == TW_TERM_ROOT) d = sm.st_s[sm.woff_s[e] + pe] - ws.ins[j];
                else d = ws.ine[j] - sm.st_e[sm.woff_e[e] + pe];
                cost = dadd(cost, term_logpdf_cold(prm.mode, prm_base, n_terms, brel, tt, sm.etab, (double)d));
              }
            }
            cost = cost + 0.0;                  // -0.0 and +0.0 are one score
            ws.ent_key[en] = score_key(cost);   // NaN -> 0
          }
        }
        __syncwarp();
      }
      TW_CPHASE(5);                                  // 2b scores
      // 2c. per-owner segments of the list (entries are grouped by owner, in leaf order)
      ws.seg_lo[lane] = 0;
      ws.seg_hi[lane] = 0;
      __syncwarp();
      for (int en = lane; en < n_ent; en += 32) {
        const int j = ws.ent_j[en];
        if (en == 0 || ws.ent_j[en - 1] != j) ws.seg_lo[j] = en;
        if (en == n_ent - 1 || ws.ent_j[en + 1] != j) ws.seg_hi[j] = en + 1;
      }
      __syncwarp();
      const int sa = ws.seg_lo[lane], sz = ws.seg_hi[lane];
      nfeas += sz - sa;
      if (has_params) {
        // An in-span whose combinations all fell into this chunk (the rule) and whose segment is
        // short is ranked by its ENTRIES in parallel: entry en counts the larger keys of its segment
        // and, if fewer than K, writes itself to that rank.  Equal keys / NaN -> the tile is redone.
        const bool whole = cneed > 0 && cstart >= chunk_base && cend <= base;
        const bool quick = whole && sz - sa <= kS3RankMax;
        ws.seg_quick[lane] = (uint8_t)quick;
        __syncwarp();
        bool bad = false;
        for (int en = lane; en < n_ent; en += 32) {
          const int j = ws.ent_j[en];
          if (!ws.seg_quick[j]) continue;
          const unsigned long long k = ws.ent_key[en];
          const int a = ws.seg_lo[j], z = ws.seg_hi[j];
          int rank = 0;
          bool tie = k == 0ull;
          for (int q = a; q < z; ++q) {
            const unsigned long long o = ws.ent_key[q];
            rank += o > k;
            tie = tie || (o == k && q != en);
          }
          bad = bad || tie;
          if (rank < TW_K) {
            ws.top_key[j][rank] = k;
            ws.top_xp[j][rank] = ws.ent_xp[en];
          }
        }
        redo = redo || bad;
        __syncwarp();
        if (quick) {
          const int len = sz - sa;
          tk0 = len > 0 ? ws.top_key[lane][0] : 0ull; tx0 = len > 0 ? ws.top_xp[lane][0] : (XP)0;
          tk1 = len > 1 ? ws.top_key[lane][1] : 0ull; tx1 = len > 1 ? ws.top_xp[lane][1] : (XP)0;
          tk2 = len > 2 ? ws.top_key[lane][2] : 0ull; tx2 = len > 2 ? ws.top_xp[lane][2] : (XP)0;
          tk3 = len > 3 ? ws.top_key[lane][3] : 0ull; tx3 = len > 3 ? ws.top_xp[lane][3] : (XP)0;
          tk4 = len > 4 ? ws.top_key[lane][4] : 0ull; tx4 = len > 4 ? ws.top_xp[lane][4] : (XP)0;
        }
        // long or streamed segments, one at a time by the WHOLE warp: every lane keeps the top K of
        // the entries a + lane, a + lane + 32, ... (the owner lane starts from its running list), then
        // K rounds of "largest head over the lanes" give the segment's top K to the owner.
        unsigned slow = __ballot_sync(kFull, !quick && sz > sa);
        while (slow) {
          const int j = __ffs(slow) - 1;
          slow &= slow - 1u;
          const int a = __shfl_sync(kFull, sa, j), z = __shfl_sync(kFull, sz, j);
          const bool own = lane == j;
          unsigned long long l0 = own ? tk0 : 0ull, l1 = own ? tk1 : 0ull, l2 = own ? tk2 : 0ull,
                             l3 = own ? tk3 : 0ull, l4 = own ? tk4 : 0ull;
          XP y0 = own ? tx0 : (XP)0, y1 = own ? tx1 : (XP)0, y2 = own ? tx2 : (XP)0, y3 = own ? tx3 : (XP)0,
             y4 = own ? tx4 : (XP)0;
          bool bad = false;
          for (int en = a + lane; en < z; en += 32) {
            unsigned long long k = ws.ent_key[en];
            if (k == 0ull) { bad = true; continue; }        // NaN score: the reference's order decides
            if (k < l4) continue;
            XP xq = ws.ent_xp[en];
            bad = bad || k == l0 || k == l1 || k == l2 || k == l3 || k == l4;   // equal keys: tie order
#define TW_S3_CE(K, X)                                              \
  if (k > K) { const unsigned long long tkk = K; K = k; k = tkk;    \
               const XP txx = X; X = xq; xq = txx; }
            TW_S3_CE(l0, y0) TW_S3_CE(l1, y1) TW_S3_CE(l2, y2) TW_S3_CE(l3, y3) TW_S3_CE(l4, y4)
#undef TW_S3_CE
          }
          unsigned long long n0 = 0, n1 = 0, n2 = 0, n3 = 0, n4 = 0;
          XP m0 = 0, m1 = 0, m2 = 0, m3 = 0, m4 = 0;
#pragma unroll
          for (int r = 0; r < TW_K; ++r) {
            const uint32_t hi = (uint32_t)(l0 >> 32);
            const uint32_t mh = __reduce_max_sync(kFull, hi);
            const uint32_t lo32 = hi == mh ? (uint32_t)l0 : 0u;
            const uint32_t ml = __reduce_max_sync(kFull, lo32);
            const unsigned long long key = ((unsigned long long)mh << 32) | ml;
            const unsigned win = __ballot_sync(kFull, key != 0ull && l0 == key);
            if (__popc(win) > 1) bad = true;                 // the same key twice: tie order
            const int wl = win ? __ffs(win) - 1 : 0;
            const XP xw = __shfl_sync(kFull, y0, wl);
            if (r == 0) { n0 = key; m0 = xw; }
            if (r == 1) { n1 = key; m1 = xw; }
            if (r == 2) { n2 = key; m2 = xw; }
            if (r == 3) { n3 = key; m3 = xw; }
            if (r == 4) { n4 = key; m4 = xw; }
            if (win && lane == wl) { l0 = l1; l1 = l2; l2 = l3; l3 = l4; l4 = 0ull; y0 = y1; y1 = y2; y2 = y3; y3 = y4; }
          }
          if (own) {
            tk0 = n0; tk1 = n1; tk2 = n2; tk3 = n3; tk4 = n4;
            tx0 = m0; tx1 = m1; tx2 = m2; tx3 = m3; tx4 = m4;
          }
          redo = redo || bad;
        }
      }
      __syncwarp();
      TW_CPHASE(6);                                  // 2c top-K
      n_ent = 0;
      if (base >= total_c) break;
    }
    if (admitted) pending = false;
  }
  if (__any_sync(kFull, redo)) {
    if (lane == 0) overflow_flag[t] = 1;       // (also under keep_windows: a score tie depends on the parameters)
    TW_CCOUNT(17, 1);                                // tie / NaN (per warp)
    return;
  }

  TW_CPHASE(2);
  // ================= results, staged through shared memory =================
  const int w0 = wid * 32;
  const int nv = min(32, cnt - w0);            // in-spans of this warp
  if (nv <= 0) return;
  const int64_t g0 = in_off + i0 + w0;
  if (worker) out.n_feasible[g0 + lane] = nfeas;
  if (has_params) {
    const int kc = (tk0 != 0) + (tk1 != 0) + (tk2 != 0) + (tk3 != 0) + (tk4 != 0);
    if (worker) out.topk_cnt[g0 + lane] = (uint8_t)kc;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    double* sd = ws.tbl;
    sd[lane * TW_K + 0] = tk0 ? key_to_score3(tk0) : nan;
    sd[lane * TW_K + 1] = tk1 ? key_to_score3(tk1) : nan;
    sd[lane * TW_K + 2] = tk2 ? key_to_score3(tk2) : nan;
    sd[lane * TW_K + 3] = tk3 ? key_to_score3(tk3) : nan;
    sd[lane * TW_K + 4] = tk4 ? key_to_score3(tk4) : nan;
    __syncwarp();
    warp_copy_out(out.topk_score + g0 * TW_K, sd, nv * TW_K * 2, lane);
    __syncwarp();
    // indices: lanes in groups that fit the staging area
    constexpr int kPer = TW_K * E;                       // ints per in-span
    constexpr int kGroup = (kS3Tbl * 2) / kPer >= 32 ? 32 : 16;
    static_assert(kS3Tbl <= 4096, "val_slot packs the slot index into 12 bits");
    static_assert((kS3Tbl * 2) / kPer >= 16, "staging area too small for the index block");
    int* si = reinterpret_cast<int*>(ws.tbl);
    int32_t* gidx = out.topk_idx + TW_K * (tuple_off + (int64_t)(i0 + w0) * E);
#pragma unroll
    for (int gq = 0; gq < 32 / kGroup; ++gq) {
      const int l0 = gq * kGroup;
      if (lane >= l0 && lane < l0 + kGroup) {
        int* row = si + (lane - l0) * kPer;
        const unsigned long long ks[TW_K] = {tk0, tk1, tk2, tk3, tk4};
        const XP xs[TW_K] = {tx0, tx1, tx2, tx3, tx4};
#pragma unroll
        for (int k = 0; k < TW_K; ++k)
#pragma unroll
          for (int e = 0; e < E; ++e)
            row[k * E + e] = ks[k] ? sm.win_a[e] + lo_get<E>(lp, e) + (int)((xs[k] >> (6 * (E - 1 - e))) & 63) : -1;
      }
      __syncwarp();
      const int nl = min(kGroup, nv - l0);
      if (nl > 0) warp_copy_out(gidx + (size_t)l0 * kPer, si, nl * kPer, lane);
      __syncwarp();
    }
  }
  if (!keep_windows && out.used_lo) {
    int* si = reinterpret_cast<int*>(ws.tbl);
#pragma unroll
    for (int e = 0; e < E; ++e) si[lane * E + e] = sm.win_a[e] + lo_get<E>(lp, e);
    __syncwarp();
    const int64_t tb = tuple_off + (int64_t)(i0 + w0) * E;
    warp_copy_out(out.used_lo + tb, si, nv * E, lane);
    warp_copy_out(out.used_bits + 2 * tb, &ws.used[0][0][0], nv * E * kNarrowW, lane);
    if (worker) out.used_wide[g0 + lane] = 0;
  }
  TW_CPHASE(7);                                      // results
}

// ---------------------------------------------------------------------------------------------
// Tile pre-pass (once per bound batch: depends on the span arrays only): the slice of every ep's
// list that holds all candidates of the tile's in-spans,
//   [lower_bound(start >= first in.start), upper_bound(start <= max in.end)).
// One warp per tile.  tile_win[t][2e] = first index, [2e+1] = length.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_tile_meta(tw_batch b, TileList tiles, int32_t* __restrict__ tile_win) {
  const int t = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= tiles.n_tiles) return;
  const int p = tiles.tile_prob[t], i0 = tiles.tile_start[t];
  const int64_t in_off = b.prob_in_off[p];
  const int n = (int)(b.prob_in_off[p + 1] - in_off);
  const int cnt = min(tiles.tile_len, n - i0);
  int64_t mx = INT64_MIN;
  for (int k = lane; k < cnt; k += 32) {
    const int64_t v = b.in_end[in_off + i0 + k];
    mx = v > mx ? v : mx;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const int64_t o = __shfl_xor_sync(kFull, mx, d);
    mx = o > mx ? o : mx;
  }
  const int ep0 = b.prob_ep_off[p];
  const int E = b.prob_ep_off[p + 1] - ep0;
  if (lane < E) {
    const int64_t off = b.ep_out_off[ep0 + lane];
    const int no = (int)(b.ep_out_off[ep0 + lane + 1] - off);
    const int a = lower_bound(b.out_start + off, no, b.in_start[in_off + i0]);
    const int z = upper_bound(b.out_start + off, no, mx);
    tile_win[(size_t)t * 2 * TW_MAX_E + 2 * lane] = a;
    tile_win[(size_t)t * 2 * TW_MAX_E + 2 * lane + 1] = z > a ? z - a : 0;
  }
}

cudaError_t launch_tile_meta(const tw_batch& b, const TileList& tiles, int32_t* tile_win, cudaStream_t s,
                             int64_t& launches) {
  if (tiles.n_tiles == 0) return cudaSuccess;
  const int blocks = (tiles.n_tiles + 3) / 4;
  k_tile_meta<<<blocks, 128, 0, s>>>(b, tiles, tile_win);
  return after_launch(launches);
}

// ---------------------------------------------------------------------------------------------
// PerfectCut(i), V3:1024-1039, from the candidate maps: cut iff the maps of prev(i) (the
// latest-ending earlier in-span, V3:1026-1032) and of i are disjoint and end(prev) <= end(i).
// One thread per in-span, CTA per tile.  Tiles redone by the sequential kernel have their flags
// written there.  A prev whose map is wide (it lives in a redone tile) is enumerated on the spot.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kS3Threads)
k_cut(tw_batch b, tw_score_out out, TileList tiles, const int32_t* __restrict__ prev_idx,
      const uint8_t* __restrict__ overflow_flag) {
  const int t = blockIdx.x;
  if (overflow_flag[t]) return;
  const int p = tiles.tile_prob[t];
  const int64_t in_off = b.prob_in_off[p];
  const int n = (int)(b.prob_in_off[p + 1] - in_off);
  const int i = tiles.tile_start[t] + threadIdx.x;
  if (i >= n || threadIdx.x >= tiles.tile_len) return;
  uint8_t cut = 0;
  if (i >= 1 && i <= n - 2) {
    const int ep0 = b.prob_ep_off[p];
    const int E = b.prob_ep_off[p + 1] - ep0;
    const int64_t tuple_off = b.prob_tuple_off[p];
    const int pi = prev_idx[in_off + i];
    bool disjoint = true;
    if (!out.used_wide[in_off + pi]) {
      for (int e = 0; e < E && disjoint; ++e) {
        const int64_t a = tuple_off + (int64_t)pi * E + e, c = tuple_off + (int64_t)i * E + e;
        if (bitmaps_intersect(out.used_bits + 2 * a, out.used_lo[a], out.used_bits + 2 * c, out.used_lo[c], kNarrowW))
          disjoint = false;
      }
    } else {
      ProbView v;
      load_view(b, p, v);
      OutWin w[TW_MAX_E];
      int lo[TW_MAX_E];
      const int64_t ps = v.is[pi], pe = v.ie[pi];
      for (int e = 0; e < E; ++e) {
        w[e].s = v.os[e]; w[e].e = v.oe[e]; w[e].base = 0; w[e].n = v.n_out[e];
        lo[e] = lower_bound(w[e].s, w[e].n, ps);
      }
      const int64_t cb = tuple_off + (int64_t)i * E;
      enumerate(v, ps, pe, w, lo, [](int, int) { return false; },
                [&](const int* c, const int64_t*, const int64_t*) {
                  for (int e = 0; e < E; ++e) {
                    const int bit = c[e] - out.used_lo[cb + e];
                    if (bit >= 0 && bit < 32 * kNarrowW && (out.used_bits[2 * (cb + e) + (bit >> 5)] >> (bit & 31) & 1u))
                      disjoint = false;
                  }
                });
    }
    cut = (uint8_t)(disjoint && b.in_end[in_off + pi] <= b.in_end[in_off + i]);
  }
  out.cut[in_off + i] = cut;
}

template <int E>
static cudaError_t setup_from() {   // k_score3<E> .. k_score3<TW_MAX_E>
  cudaError_t e = cudaFuncSetAttribute(k_score3<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(S3Smem<E>));
  if constexpr (E < TW_MAX_E) {
    if (e == cudaSuccess) e = setup_from<E + 1>();
  }
  return e;
}

cudaError_t setup_score3() { return setup_from<1>(); }

template <int E>
static cudaError_t launch_one(const tw_batch& b, const tw_params& prm, int has_params, int keep, const tw_score_out& out,
                              const TileList& tl, const int32_t* tile_win, uint8_t* ovf, cudaStream_t s,
                              int64_t& launches) {
  k_score3<E><<<tl.n_tiles, kS3Threads, sizeof(S3Smem<E>), s>>>(b, prm, has_params, keep, out, tl, tile_win, ovf);
  return after_launch(launches);
}

cudaError_t launch_score3(const tw_batch& b, const tw_params* prm, const tw_score_out& out, int keep_windows,
                          const ScoreTiles& st, const int32_t* prev_idx, cudaStream_t s, int64_t& launches) {
  tw_params dummy;
  dummy.mode = TW_PARAMS_MIXTURE; dummy.reserved0 = 0;
  dummy.prob_gauss_off = nullptr; dummy.gauss = nullptr; dummy.mix = nullptr;
  const tw_params& pr = prm ? *prm : dummy;
  const int hp = prm != nullptr;
  cudaError_t e = cudaSuccess;
  if (!keep_windows) {
    e = cudaMemsetAsync(st.overflow, 0, (size_t)st.n_tiles, s);
    if (e != cudaSuccess) return e;
  }
  for (int E = 1; E <= TW_MAX_E; ++E) {
    const int c0 = st.class_off[E - 1], c1 = st.class_off[E];
    if (c1 == c0) continue;
    TileList tl{st.tile_prob + c0, st.tile_start + c0, c1 - c0, kS3Tile};
    const int32_t* twin = st.tile_win + (size_t)c0 * 2 * TW_MAX_E;
    uint8_t* ovf = st.overflow + c0;
    switch (E) {
      case 1: e = launch_one<1>(b, pr, hp, keep_windows, out, tl, twin, ovf, s, launches); break;
      case 2: e = launch_one<2>(b, pr, hp, keep_windows, out, tl, twin, ovf, s, launches); break;
      case 3: e = launch_one<3>(b, pr, hp, keep_windows, out, tl, twin, ovf, s, launches); break;
      case 4: e = launch_one<4>(b, pr, hp, keep_windows, out, tl, twin, ovf, s, launches); break;
      case 5: e = launch_one<5>(b, pr, hp, keep_windows, out, tl, twin, ovf, s, launches); break;
      case 6: e = launch_one<6>(b, pr, hp, keep_windows, out, tl, twin, ovf, s, launches); break;
      case 7: e = launch_one<7>(b, pr, hp, keep_windows, out, tl, twin, ovf, s, launches); break;
      default: e = launch_one<8>(b, pr, hp, keep_windows, out, tl, twin, ovf, s, launches); break;
    }
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t launch_cut(const tw_batch& b, const tw_score_out& out, const ScoreTiles& st, const int32_t* prev_idx,
                       cudaStream_t s, int64_t& launches) {
  TileList tl{st.tile_prob, st.tile_start, st.n_tiles, kS3Tile};
  k_cut<<<st.n_tiles, kS3Threads, 0, s>>>(b, out, tl, prev_idx, st.overflow);
  return after_launch(launches);
}

}  // namespace tw
