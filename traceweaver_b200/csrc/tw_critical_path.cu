// tw_critical_path.cu — critical paths of the reconstructed requests (tw_critical_paths).
//
// After the join (tw_traces.cu) every request is a tree of nodes.  Windows are handed down the trees one
// level of in-spans per launch: a thread takes an on-path in-span, chooses which of its out-spans are on
// the path (cp_in_span_step, tw_core.cuh), and for each of them whether the callee's in-span is
// (cp_out_span_step), whose window it writes for the next level.  The last level walks everything below
// its in-spans itself, without a stack (cp_tail_walk), so no result depends on how many levels were
// launched.  Then every request's culprit, by an integer max over the bits of the (non-negative) self
// times and a min over the node ids that hold it, and the per-service sums, one CTA per service or callee
// in a fixed order.  No float atomics: every result is the same from run to run, for any grid and any
// level count.
#include "tw_kernels.cuh"

namespace tw {

namespace {

template <class T>
struct CpTimes {
  const T* in_s;
  const T* in_e;
  const T* out_s;
  const T* out_e;
};

// In-span x on the path with window [a, b]: its self time, its chosen out-spans' self times, and the
// windows of the callee in-spans that go on the path, whose level words become `mark` (returns their
// count).
template <class T>
__device__ int cp_visit(const tw_batch& bt, const CpTimes<T>& t, const int32_t* __restrict__ assign,
                        const int32_t* __restrict__ claim, const tw_critical_out& out, T* wlo, T* whi,
                        int32_t* level, int32_t x, T a, T b, int mark) {
  const int32_t n_in = (int32_t)bt.n_in_total;
  const int p = last_le(bt.prob_in_off, bt.n_problems, x);
  const int64_t in0 = bt.prob_in_off[p], n = bt.prob_in_off[p + 1] - in0, i = x - in0;
  const int ep0 = bt.prob_ep_off[p], E = bt.prob_ep_off[p + 1] - ep0;
  bool has[TW_MAX_E], on[TW_MAX_E];
  T cs[TW_MAX_E], ce[TW_MAX_E], lo[TW_MAX_E], hi[TW_MAX_E];
  int32_t k[TW_MAX_E];
  for (int e = 0; e < E; ++e) {
    const int32_t j = assign[bt.prob_tuple_off[p] + e * n + i];
    has[e] = j >= 0;                                 // in range: the join checked it
    k[e] = has[e] ? (int32_t)(bt.ep_out_off[ep0 + e] + j) : 0;
    cs[e] = has[e] ? t.out_s[k[e]] : T(0);
    ce[e] = has[e] ? t.out_e[k[e]] : T(0);
  }
  const T self = cp_in_span_step<T>(E, has, cs, ce, a, b, on, lo, hi);
  out.on_path[x] = 1;
  out.self_us[x] = (double)self;
  int m = 0;
  for (int e = 0; e < E; ++e) {
    if (!on[e]) continue;
    const int32_t y = claim[k[e]];
    bool y_on = false;
    T ylo = 0, yhi = 0;
    const T ks = cp_out_span_step<T>(lo[e], hi[e], y >= 0, y >= 0 ? t.in_s[y] : T(0), y >= 0 ? t.in_e[y] : T(0),
                                     &y_on, &ylo, &yhi);
    out.on_path[n_in + k[e]] = 1;
    out.self_us[n_in + k[e]] = (double)ks;
    if (y_on) {
      wlo[y] = ylo;
      whi[y] = yhi;
      level[y] = mark;
      ++m;
    }
  }
  return m;
}

// The trees below the last level L for cp_tail_walk (tw_core.cuh): children through `assign` and the
// caller-claim words, marked when their level word is L + 1; parents through the join's parent words.
template <class T>
struct CpTail {
  const tw_batch& bt;
  const CpTimes<T>& t;
  const int32_t* __restrict__ assign;
  const int32_t* __restrict__ claim;
  const int32_t* __restrict__ parent;
  const tw_critical_out& out;
  const CpScratch& sc;
  int mark;
  int64_t tup, n, i;                             // the entered in-span: its service's tuples, size, own index
  int ep0;                                       // and the service's first global callee

  __device__ int enter(int32_t y) {
    const int p = last_le(bt.prob_in_off, bt.n_problems, y);
    const int64_t in0 = bt.prob_in_off[p];
    tup = bt.prob_tuple_off[p];
    n = bt.prob_in_off[p + 1] - in0;
    i = y - in0;
    ep0 = bt.prob_ep_off[p];
    return bt.prob_ep_off[p + 1] - ep0;
  }
  __device__ int32_t child(int e) const {
    const int32_t j = assign[tup + e * n + i];
    if (j < 0) return -1;
    const int32_t y = claim[bt.ep_out_off[ep0 + e] + j];
    return y >= 0 && sc.level[y] == mark ? y : -1;
  }
  __device__ void visit(int32_t y) {
    T* wlo = (T*)sc.wlo;
    T* whi = (T*)sc.whi;
    cp_visit<T>(bt, t, assign, claim, out, wlo, whi, sc.level, y, wlo[y], whi[y], mark);
  }
  __device__ int32_t up(int32_t y, int* e) const {
    const int32_t k = parent[y];                 // y's caller: out-span node n_in + its index
    const int32_t x = parent[k];
    const int ep = last_le(bt.ep_out_off, bt.n_ep_total, (int64_t)k - bt.n_in_total);
    *e = ep - bt.prob_ep_off[last_le(bt.prob_in_off, bt.n_problems, x)];
    return x;
  }
};

// Level L: one thread per in-span walked at L (level 0: the request roots, whose windows are their own
// intervals).  The in-spans it puts on the path are walked at L + 1.  A level after one that put nothing
// on the path returns at once.  The last level (`last`) walks what lies below its in-spans itself
// (cp_tail_walk), at any depth.  Level 0 also sets culprit[] to INT_MAX for a root and -1 otherwise, flags
// the slow requests and counts the requests.
template <class T>
__global__ void __launch_bounds__(kTreeThreads)
k_cp_level(tw_batch bt, CpTimes<T> t, const int32_t* __restrict__ assign, const int32_t* __restrict__ claim,
           const int32_t* __restrict__ parent, tw_critical_out out, CpScratch sc, int L, int last, double slow_us) {
  if (L > 0 && *(volatile int*)&sc.act[L - 1] == 0) return;
  const int64_t n_in = bt.n_in_total;
  T* wlo = (T*)sc.wlo;
  T* whi = (T*)sc.whi;
  bool activated = false;
  int n_req = 0, n_slow = 0;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_in; g += (int64_t)gridDim.x * blockDim.x) {
    const int32_t x = (int32_t)g;
    T a, b;
    if (L == 0) {
      const bool is_root = out.root[x] == x;
      out.culprit[x] = is_root ? 0x7fffffff : -1;
      if (!is_root) continue;
      a = t.in_s[x];
      const T e = t.in_e[x];
      b = e > a ? e : a;
      const bool slow = (double)(b - a) >= slow_us;
      sc.slow[x] = slow;
      ++n_req;
      n_slow += slow;
    } else {
      if (sc.level[x] != L) continue;
      a = wlo[x];
      b = whi[x];
    }
    const int m = cp_visit<T>(bt, t, assign, claim, out, wlo, whi, sc.level, x, a, b, L + 1);
    activated |= m > 0;
    if (last && m > 0) {
      CpTail<T> g{bt, t, assign, claim, parent, out, sc, L + 1};
      cp_tail_walk(g, x);
    }
  }
  if (__syncthreads_or(activated) && threadIdx.x == 0) sc.act[L] = 1;
  if (L == 0) {
    n_req = __reduce_add_sync(0xffffffffu, n_req);
    n_slow = __reduce_add_sync(0xffffffffu, n_slow);
    if ((threadIdx.x & 31) == 0 && n_req) {
      atomicAdd(&out.requests[0], n_req);
      if (n_slow) atomicAdd(&out.requests[1], n_slow);
    }
  }
}

// cmax[r]: the largest self-time bits over the on-path nodes of request r (non-negative doubles order as
// their bits)
__global__ void __launch_bounds__(kTreeThreads)
k_cp_culprit_max(int64_t n_nodes, const uint8_t* __restrict__ on_path, const int32_t* __restrict__ root,
                 const double* __restrict__ self, unsigned long long* __restrict__ cmax) {
  for (int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; x < n_nodes; x += (int64_t)gridDim.x * blockDim.x)
    if (on_path[x]) atomicMax(&cmax[root[x]], (unsigned long long)__double_as_longlong(self[x]));
}

// culprit[r]: the smallest on-path node of request r whose self time is cmax[r]
__global__ void __launch_bounds__(kTreeThreads)
k_cp_culprit_min(int64_t n_nodes, const uint8_t* __restrict__ on_path, const int32_t* __restrict__ root,
                 const double* __restrict__ self, const unsigned long long* __restrict__ cmax,
                 int32_t* __restrict__ culprit) {
  for (int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; x < n_nodes; x += (int64_t)gridDim.x * blockDim.x) {
    if (!on_path[x]) continue;
    const int32_t r = root[x];
    if ((unsigned long long)__double_as_longlong(self[x]) == cmax[r]) atomicMin(&culprit[r], (int32_t)x);
  }
}

// One CTA per segment: services p < P (their in-span nodes), then callees ep (their out-span nodes), each
// summed in tree_cta_sum's fixed order: column 0 all on-path nodes, column 1 those of slow requests.
__global__ void __launch_bounds__(kTreeThreads)
k_cp_reduce(tw_batch bt, const uint8_t* __restrict__ slow, tw_critical_out out) {
  __shared__ double ws[2][kTreeThreads / 32];
  __shared__ int wc[2][kTreeThreads / 32];
  const int P = bt.n_problems, n_seg = P + bt.n_ep_total;
  for (int sg = blockIdx.x; sg < n_seg; sg += gridDim.x) {
    int64_t lo, hi;
    if (sg < P) {
      lo = bt.prob_in_off[sg];
      hi = bt.prob_in_off[sg + 1];
    } else {
      lo = bt.n_in_total + bt.ep_out_off[sg - P];
      hi = bt.n_in_total + bt.ep_out_off[sg - P + 1];
    }
    double s[2];
    int c[2];
    tree_cta_sum(lo, hi, [&](int64_t x, double* a, int* k) {
      if (!out.on_path[x]) return;
      const double v = out.self_us[x];
      a[0] = dadd(a[0], v);
      ++k[0];
      if (slow[out.root[x]]) {
        a[1] = dadd(a[1], v);
        ++k[1];
      }
    }, ws, wc, s, c);
    if (threadIdx.x == 0) {
      if (sg < P) {
        out.server_us[2 * sg] = s[0];
        out.server_us[2 * sg + 1] = s[1];
        out.server_visits[2 * sg] = c[0];
        out.server_visits[2 * sg + 1] = c[1];
      } else {
        out.call_us[2 * (sg - P)] = s[0];
        out.call_us[2 * (sg - P) + 1] = s[1];
      }
    }
  }
}

template <class T>
cudaError_t launch_walk(const tw_batch& b, const CpTimes<T>& t, const int32_t* assign, const int32_t* claim,
                        const int32_t* parent, double slow_us, const tw_critical_out& out, const CpScratch& sc,
                        int levels, int n_sm, cudaStream_t s, int64_t& launches) {
  const unsigned g = tree_grid(b.n_in_total, n_sm);
  for (int L = 0; L < levels; ++L) {
    k_cp_level<T><<<g, kTreeThreads, 0, s>>>(b, t, assign, claim, parent, out, sc, L, L == levels - 1, slow_us);
    const cudaError_t e = after_launch(launches);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace

cudaError_t launch_critical_paths(const tw_batch& b, const tw_times_f64* f64, const int32_t* assign,
                                  const int32_t* claim, const int32_t* parent, double slow_us,
                                  const tw_critical_out& out, const CpScratch& sc, int levels, int n_sm,
                                  cudaStream_t s, int64_t& launches) {
  const int64_t n_in = b.n_in_total, n_nodes = n_in + b.n_out_total;
  cudaError_t e;
  if ((e = cudaMemsetAsync(out.on_path, 0, (size_t)n_nodes, s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(out.self_us, 0, (size_t)n_nodes * sizeof(double), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(out.requests, 0, 2 * sizeof(int32_t), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(sc.level, 0xff, (size_t)n_in * sizeof(int32_t), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(sc.cmax, 0, (size_t)n_in * sizeof(unsigned long long), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(sc.act, 0, (size_t)levels * sizeof(int), s)) != cudaSuccess) return e;
  if (f64)
    e = launch_walk<double>(b, CpTimes<double>{f64->in_start, f64->in_end, f64->out_start, f64->out_end}, assign,
                            claim, parent, slow_us, out, sc, levels, n_sm, s, launches);
  else
    e = launch_walk<int64_t>(b, CpTimes<int64_t>{b.in_start, b.in_end, b.out_start, b.out_end}, assign, claim,
                             parent, slow_us, out, sc, levels, n_sm, s, launches);
  if (e != cudaSuccess) return e;
  const unsigned g = tree_grid(n_nodes, n_sm);
  k_cp_culprit_max<<<g, kTreeThreads, 0, s>>>(n_nodes, out.on_path, out.root, out.self_us, sc.cmax);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  k_cp_culprit_min<<<g, kTreeThreads, 0, s>>>(n_nodes, out.on_path, out.root, out.self_us, sc.cmax, out.culprit);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  const int64_t n_seg = (int64_t)b.n_problems + b.n_ep_total;
  const int64_t cap = (int64_t)n_sm * 8;
  k_cp_reduce<<<(unsigned)(n_seg < cap ? n_seg : cap), kTreeThreads, 0, s>>>(b, sc.slow, out);
  return after_launch(launches);
}

}  // namespace tw
