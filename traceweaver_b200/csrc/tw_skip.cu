// tw_skip.cu — skip / cache mode (SURVEY.md §8 rows a11, a12, f-4): services whose outgoing lists do
// not have one span per incoming span (overall_skip_budget != 0, traceweaver_v3.py:1138-1158).
//
// Replaces, for such a service (reference: .../algorithms/traceweaver_v3.py = V3, traceweaver_v1.py = V1)
//   CreateWindows2 on the lists as the caller hands them over     V3:1020-1078 (FindCutoffs :182-217
//       literally — halving searches on possibly unsorted lists, negative-index wrap — DfsTraverse3 :236-288)
//   FetchSkipFromWindow                                            V3:820-842
//   FindTopKAssignments, DfsTraverseX with the skip branch         V3:219-234, :292-351
//   ScoreAssignmentAsPerInvocationGraph with skip spans            V1:259-361 (FindValidAncestor :264-292,
//       normalised = mean of densities when a budget is positive, V3:222-227)
//   the ONE iteration of the hot loop                              V3:1155-1156, :1159-1219
//   BuildMISInstance + exact MWIS, AddAssignment / AddTopKAssignments   V3:1252-1281, V1:433-488
//   the parent search of BuildDistributions                        V3:108-172 (k_build_dist)
// The host mirror (traceweaver_b200/skipmode.py) supplies what the reference computes with NumPy
// library calls whose tie behaviour is part of the result: the water-filled skip counts
// (np.argsort, V3:884) and np.mean / np.std of the BuildDistributions samples.
//
// Mapping.  The mode is rare (exps/exp2: ONE service per run) and sequential by construction: which
// skip span a tuple receives depends on how many skip spans every earlier search has fetched
// (FetchSkipFromWindow hands out the least-used one = round robin), and deletion couples the
// windows.  One warp per service; lane 0 walks the in-spans, the other lanes only help with the
// bitmap work.  Exactness before speed: this is the path that makes `n_out != n_in` a supported
// input instead of TW_ERR_UNSUPPORTED, not a throughput path.
#include "tw_kernels.cuh"
#include "tw_skip_core.cuh"

namespace tw {

__global__ void __launch_bounds__(32)
k_skip(tw_batch b, tw_skip_desc sd, tw_skip_out out, uint32_t* __restrict__ taken,
       uint32_t* __restrict__ set_scratch, const int64_t* __restrict__ prob_set_off,
       int32_t* __restrict__ win_scratch, long long node_limit, int* __restrict__ err_flag) {
  __shared__ SkipShared sh;
  if (threadIdx.x != 0) return;        // (sequential by construction, see the file header)
  const int rc = skip_solve_problem(b, blockIdx.x, sd, out, taken, set_scratch, prob_set_off, win_scratch, node_limit, sh);
  if (rc != TW_OK) atomicMin(err_flag, rc);
}

cudaError_t launch_skip(const tw_batch& b, const tw_skip_desc& sd, const tw_skip_out& out, uint32_t* taken,
                        uint32_t* set_scratch, const int64_t* prob_set_off, int32_t* win_scratch,
                        long long node_limit, int* err_flag, cudaStream_t s, int64_t& launches) {
  k_skip<<<b.n_problems, 32, 0, s>>>(b, sd, out, taken, set_scratch, prob_set_off, win_scratch, node_limit, err_flag);
  return after_launch(launches);
}

// ---------------------------------------------------------------------------------------------
// BuildDistributions' parent search (V3:120-168) over the service's spans merged by start (stable,
// incoming spans first, then the out eps in topological order — the host mirror merges).  One thread
// per span: the nearest preceding span that qualifies as its parent within large_delay.
//   label 0 = server span (incoming), 1 + e = client span of out ep e.
//   key[i] = parent_label * (E + 1) + label, or -1;  val[i] = the delay sample.
// ---------------------------------------------------------------------------------------------
__global__ void k_build_dist(int n, const int64_t* __restrict__ ms, const int64_t* __restrict__ me,
                             const int8_t* __restrict__ label, int E, int64_t large_delay,
                             int32_t* __restrict__ key, int64_t* __restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t s = ms[i], e = me[i];
  const int lab = label[i];
  int k = -1;
  int64_t vv = 0;
  for (int j = i - 1; j >= 0; --j) {
    const int64_t ps = ms[j], pe = me[j];
    if (e - ps > large_delay) break;                        // V3:126, :152
    const int pl = label[j];
    if (lab != 0) {                                          // client span
      if (pl == 0) { k = pl * (E + 1) + lab; vv = s - ps; break; }                    // V3:128-131, :141
      if (pe < s && pl < lab) { k = pl * (E + 1) + lab; vv = s - pe; break; }          // V3:132-137, :143
    } else if (pl != 0 && pe < e) {                          // server span, client parent, V3:154-163
      k = pl * (E + 1) + lab; vv = e - pe; break;
    }
  }
  key[i] = k;
  val[i] = vv;
}

cudaError_t launch_build_dist(int n, const int64_t* ms, const int64_t* me, const int8_t* label, int E,
                              int64_t large_delay, int32_t* key, int64_t* val, cudaStream_t s, int64_t& launches) {
  if (n <= 0) return cudaSuccess;
  k_build_dist<<<(n + 127) / 128, 128, 0, s>>>(n, ms, me, label, E, large_delay, key, val);
  return after_launch(launches);
}

}  // namespace tw
