// tw_traces.cu — end-to-end request trees from the per-service assignments (tw_assemble_traces).
//
// Replaces (reference: src/trace_reconstructor/ports/python/)
//   ConstructEndToEndTraces               helpers/utils.py:216, called from executor.py:1210-1230
// The reference walks its per-service maps span by span.  Here a batch's spans are nodes of one forest
// (in-spans [0, n_in), out-spans n_in + [0, n_out)): the predicted links (assign: in-span -> out-span) and
// the observed ones (in_caller: in-span -> the client span of its RPC) are scattered into a parent array,
// every node finds its root by pointer jumping, and the roots count their nodes.  All integer work: the
// result does not depend on the order in which threads run.
#include "tw_kernels.cuh"

namespace tw {

namespace {

// One thread per tuple (problem p, callee e, in-span i): assign = j >= 0 makes in-span i the parent of
// out-span j of callee e.  parent[] of the out-spans starts at -1 and is the claim word: a second claim
// finds it taken.  err[0]: smallest out-span node claimed twice; err[2]: smallest in-span node with an
// index outside its callee's list.
__global__ void k_link_out(tw_batch b, const int32_t* __restrict__ assign, int32_t* __restrict__ parent,
                           int32_t* __restrict__ err) {
  const int64_t n_tuple = b.prob_tuple_off[b.n_problems];
  const int32_t n_in = (int32_t)b.n_in_total;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_tuple; g += (int64_t)gridDim.x * blockDim.x) {
    const int32_t j = assign[g];
    if (j < 0) continue;                                   // NA (-1) or a skip span (<= -2): no child
    const int p = last_le(b.prob_tuple_off, b.n_problems, g);
    const int64_t in0 = b.prob_in_off[p];
    const int64_t n = b.prob_in_off[p + 1] - in0;
    const int64_t local = g - b.prob_tuple_off[p];
    const int ep = b.prob_ep_off[p] + (int)(local / n);
    const int32_t in_node = (int32_t)(in0 + local % n);
    const int64_t o0 = b.ep_out_off[ep];
    if (j >= b.ep_out_off[ep + 1] - o0) {
      atomicMin(&err[2], in_node);
      continue;
    }
    const int32_t x = n_in + (int32_t)(o0 + j);
    if (atomicCAS(&parent[x], -1, in_node) != -1) atomicMin(&err[0], x);
  }
}

// One thread per in-span: its parent is its caller (observed).  claim[] (one word per out-span, -1) is
// taken by the first in-span naming that caller.  err[1]: smallest caller named twice; err[3]: smallest
// in-span node whose caller is neither -1 nor an out-span node.
__global__ void k_link_in(int32_t n_in, int32_t n_nodes, const int32_t* __restrict__ in_caller,
                          int32_t* __restrict__ parent, int32_t* __restrict__ claim, int32_t* __restrict__ err) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_in; k += (int64_t)gridDim.x * blockDim.x) {
    int32_t c = in_caller[k];
    if (c != -1) {
      if (c < n_in || c >= n_nodes) {
        atomicMin(&err[3], (int32_t)k);
        c = -1;
      } else if (atomicCAS(&claim[c - n_in], -1, (int32_t)k) != -1) {
        atomicMin(&err[1], c);
      }
    }
    parent[k] = c;
  }
}

// One round of pointer jumping, anc[x] <- anc[anc[x]], in place (a value read while another thread
// rewrites it is an ancestor either way).  A root is its own ancestor.  Round 0 starts from the parents:
// anc[x] = up(up(x)), up(x) = parent[x] or x for a root.  changed[r] is set when round r moved some node;
// a round after one that moved nothing returns at once, so the rounds that run are the tree depth's log.
__global__ void k_jump(int32_t n_nodes, int round, const int32_t* __restrict__ parent, int32_t* anc,
                       int* __restrict__ changed) {
  if (round > 0 && *(volatile int*)&changed[round - 1] == 0) return;
  bool moved = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_nodes; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t x = (int32_t)i;
    if (round == 0) {
      const int32_t p = parent[x];
      const int32_t a = p < 0 ? x : p;
      const int32_t pa = parent[a];
      anc[x] = pa < 0 ? a : pa;
      moved |= p >= 0;
    } else {
      const int32_t a = anc[x];
      const int32_t aa = anc[a];
      if (aa != a) {
        anc[x] = aa;
        moved = true;
      }
    }
  }
  if (__syncthreads_or(moved) && threadIdx.x == 0) changed[round] = 1;
}

// root[x] = its final ancestor if that has no parent, else -1 (x sits on or under a cycle); every root
// counts its nodes.  root[] holds the ancestors on entry.
__global__ void k_roots(int32_t n_nodes, const int32_t* __restrict__ parent, int32_t* __restrict__ root,
                        int32_t* __restrict__ size) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_nodes; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t x = (int32_t)i;
    const int32_t a = root[x];
    const int32_t r = parent[a] < 0 ? a : -1;
    root[x] = r;
    if (r >= 0) atomicAdd(&size[r], 1);
  }
}

}  // namespace

int trace_rounds(int64_t n_nodes) {
  int r = 0;
  while (((int64_t)1 << r) < n_nodes) ++r;                 // ceil(log2 n_nodes)
  return r + 1;
}

cudaError_t launch_assemble_traces(const tw_batch& b, int64_t n_tuple, const int32_t* assign, const int32_t* in_caller,
                                   int32_t* parent, int32_t* root, int32_t* size, int32_t* claim, int32_t* err,
                                   int* changed, int rounds, int n_sm, cudaStream_t s, int64_t& launches) {
  const int32_t n_in = (int32_t)b.n_in_total, n_out = (int32_t)b.n_out_total, n_nodes = n_in + n_out;
  cudaError_t e;
  if ((e = cudaMemsetAsync(parent + n_in, 0xff, (size_t)n_out * sizeof(int32_t), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(claim, 0xff, (size_t)n_out * sizeof(int32_t), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(err, 0x7f, 4 * sizeof(int32_t), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(changed, 0, (size_t)rounds * sizeof(int), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(size, 0, (size_t)n_nodes * sizeof(int32_t), s)) != cudaSuccess) return e;
  k_link_out<<<tree_grid(n_tuple, n_sm), kTreeThreads, 0, s>>>(b, assign, parent, err);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  k_link_in<<<tree_grid(n_in, n_sm), kTreeThreads, 0, s>>>(n_in, n_nodes, in_caller, parent, claim, err);
  if ((e = after_launch(launches)) != cudaSuccess) return e;
  const unsigned g = tree_grid(n_nodes, n_sm);
  for (int r = 0; r < rounds; ++r) {
    k_jump<<<g, kTreeThreads, 0, s>>>(n_nodes, r, parent, root, changed);
    if ((e = after_launch(launches)) != cudaSuccess) return e;
  }
  k_roots<<<g, kTreeThreads, 0, s>>>(n_nodes, parent, root, size);
  return after_launch(launches);
}

}  // namespace tw
