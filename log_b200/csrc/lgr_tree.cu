// Level-of-Gaussian tree traversal (SURVEY.md 8(f) row 2): TensorTree.traverse / _query_tree_torch of the reference
// (LoG/model/tensor_tree.py:132-186) together with the per-level compute_radius calls it makes
// (LoG/model/level_of_gaussian.py:64-93: gather, exp / normalize activations, compute_radius_cuda) -- as
// level-synchronous kernels that never return to the host between levels.
//
// Reference semantics reproduced exactly, including the ORDER of the returned indices (they index the gathered
// parameter arrays, point_id_pixel refers to that order):
//   level 0 : every root r: keep if radius2d(r) < min_px or r has no children, else descend
//   level l : candidates = the children (tree[node_index[parent]][c], c ascending, != -1) of the descending nodes, in
//             parent order; keep a candidate if radius2d < min_px or it is a leaf, else descend
//   cut-off : after max(1, ...) .. min(max_level, max_depth) child levels the still-descending nodes are kept as they are
//   result  : [kept roots | kept level-1 | kept level-2 | ... | cut-off nodes], each group in candidate order
//
// Three kernels per level, all with a fixed grid and grid-stride loops over a candidate count that lives on the device:
//   classify  one thread per candidate slot: gather id, radius (activations fused), keep / descend flag, per-chunk counts
//   scan      one CTA: exclusive scan of the chunk counts, advances the output offset and the next frontier size
//   scatter   stable compaction (chunk prefix + ballot rank) into the output and into the next frontier
// Levels past the actual depth find an empty frontier and exit at once; the host reads the final count once.
#include "lgr_common.cuh"
#include "lgr_prof.cuh"

namespace lgr {

constexpr int TREE_THREADS = 256;
#ifndef LGR_TREE_GRID
#define LGR_TREE_GRID 528               // 4 CTAs per SM on the 132 SMs of an H100 SXM; grid-stride loops cover any size
#endif
constexpr int TREE_GRID = LGR_TREE_GRID;


// state[0] frontier size   state[1] output size   state[2] kept (this level)   state[3] descending (this level)
constexpr int ST_FRONT = 0, ST_OUT = 1;

__device__ __forceinline__ float node_radius(const TreeArgs& a, int id, const float* sV, const float* sP) {
  float p[3];
  p[0] = __ldg(a.xyz + 3 * (int64_t)id); p[1] = __ldg(a.xyz + 3 * (int64_t)id + 1); p[2] = __ldg(a.xyz + 3 * (int64_t)id + 2);
  if (!ndc_inside(p, sP)) return 0.0f;
  float s[3];
#pragma unroll
  for (int k = 0; k < 3; k++) s[k] = expf(__ldg(a.scaling_raw + 3 * (int64_t)id + k));
  float inv;
  const float4 q = act_normalize(ldg4(a.rotation_raw + 4 * (int64_t)id), inv);
  return projected_radius(p, s, q, sV, a.fx, a.fy, a.tanfovx, a.tanfovy);
}

// flags: bit0 = keep, bit1 = descend; cand[slot] = point id of the slot (-1: empty child slot)
template <bool ROOT>
__global__ void __launch_bounds__(TREE_THREADS)
tree_classify_kernel(TreeArgs a, const int64_t* __restrict__ roots, const int32_t* __restrict__ front,
                     const int32_t* __restrict__ state, int32_t* __restrict__ cand, uint8_t* __restrict__ flags,
                     int32_t* __restrict__ chunk_cnt) {
  __shared__ float sV[16], sP[16];
  if (threadIdx.x < 16) { sV[threadIdx.x] = a.view[threadIdx.x]; sP[threadIdx.x] = a.proj[threadIdx.x]; }
  __syncthreads();
  const int64_t nslots = (int64_t)state[ST_FRONT] * (ROOT ? 1 : a.C);
  const int64_t nchunks = (nslots + TREE_THREADS - 1) / TREE_THREADS;
  for (int64_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    const int64_t slot = chunk * TREE_THREADS + threadIdx.x;
    int id = -1;
    if (slot < nslots) {
      if (ROOT) id = (int)roots[slot];
      else {
        const int parent = front[slot / a.C];
        id = a.tree[(int64_t)a.node_index[parent] * a.C + (int)(slot % a.C)];
      }
    }
    bool keep = false, next = false;
    if (id >= 0) {
      const bool leaf = a.node_index[id] == -1;
      const bool small = node_radius(a, id, sV, sP) < a.min_px;
      keep = small || leaf;
      next = !keep;
    }
    if (slot < nslots) { cand[slot] = id; flags[slot] = (uint8_t)((keep ? 1 : 0) | (next ? 2 : 0)); }
    const int nk = __syncthreads_count(keep), nn = __syncthreads_count(next);
    if (threadIdx.x == 0) { chunk_cnt[2 * chunk] = nk; chunk_cnt[2 * chunk + 1] = nn; }
  }
}

// exclusive scan of the (kept, descending) chunk counts in place; totals into state[2], state[3]
__global__ void __launch_bounds__(1024)
tree_scan_kernel(int C_or_one, int32_t* __restrict__ state, int32_t* __restrict__ chunk_cnt) {
  const int64_t nslots = (int64_t)state[ST_FRONT] * C_or_one;
  const ScanTotals<2> t = cta_exclusive_scan<1024, 2>((int)((nslots + TREE_THREADS - 1) / TREE_THREADS),
                                                      [&](int b, int k) { return chunk_cnt[2 * b + k]; },
                                                      [&](int b, int k, int pre) { chunk_cnt[2 * b + k] = pre; });
  if (threadIdx.x == 0) { state[2] = t.v[0]; state[3] = t.v[1]; }
}

// stable compaction: kept candidates append to `out`, descending ones form the next frontier
__global__ void __launch_bounds__(TREE_THREADS)
tree_scatter_kernel(int C_or_one, const int32_t* __restrict__ state, const int32_t* __restrict__ cand,
                    const uint8_t* __restrict__ flags, const int32_t* __restrict__ chunk_pre, int64_t* __restrict__ out,
                    int32_t* __restrict__ next_front) {
  __shared__ __align__(16) int wk[TREE_THREADS / 32];
  __shared__ __align__(16) int wn[TREE_THREADS / 32];
  const int64_t nslots = (int64_t)state[ST_FRONT] * C_or_one;
  const int64_t nchunks = (nslots + TREE_THREADS - 1) / TREE_THREADS;
  const int64_t out_base = state[ST_OUT];
  for (int64_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    const int64_t slot = chunk * TREE_THREADS + threadIdx.x;
    const int f = slot < nslots ? flags[slot] : 0;
    const int rk = cta_ballot_rank<TREE_THREADS>(f & 1, wk).rank, rn = cta_ballot_rank<TREE_THREADS>(f & 2, wn).rank;
    if (f & 1) out[out_base + chunk_pre[2 * chunk] + rk] = cand[slot];
    if (f & 2) next_front[chunk_pre[2 * chunk + 1] + rn] = cand[slot];
  }
}

// after scatter: the output grew by the kept candidates, the descending ones are the new frontier
__global__ void tree_advance_kernel(int32_t* __restrict__ state) {
  state[ST_OUT] += state[2];
  state[ST_FRONT] = state[3];
}

// cut-off: the still-descending nodes are returned as they are (tensor_tree.py:137-140)
__global__ void __launch_bounds__(TREE_THREADS)
tree_append_kernel(const int32_t* __restrict__ state, const int32_t* __restrict__ front, int64_t* __restrict__ out) {
  const int n = state[ST_FRONT];
  const int64_t base = state[ST_OUT];
  for (int64_t i = (int64_t)blockIdx.x * TREE_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * TREE_THREADS)
    out[base + i] = front[i];
}

__global__ void tree_finish_kernel(int32_t* __restrict__ state, int64_t* __restrict__ count_out) {
  state[ST_OUT] += state[ST_FRONT];
  state[ST_FRONT] = 0;
  *count_out = state[ST_OUT];
}

// num_roots_d: the root count on the device (the walk of lgr_prepare_select), else num_roots
__global__ void tree_init_kernel(int32_t* __restrict__ state, int num_roots, const int64_t* __restrict__ num_roots_d) {
  state[ST_FRONT] = num_roots_d ? (int)*num_roots_d : num_roots; state[ST_OUT] = 0; state[2] = 0; state[3] = 0;
}

// scratch layout (int32 units): state[8] | front A [P] | front B [P] | cand [S] | chunk counts [2 * ceil(S/256) + 2] |
// flags [S bytes], with P = num_points, S = max(num_roots, num_nodes * C) candidate slots of one level.  num_roots_d: the
// number of roots lives on the device (at most num_roots, which then only sizes the scratch).
int launch_tree_traverse(const TreeArgs& a, int64_t num_points, int64_t num_nodes, const int64_t* roots, int64_t num_roots,
                         const int64_t* num_roots_d, int levels, int32_t* scratch, int64_t* out, int64_t* count_out,
                         cudaStream_t st) {
  const int64_t S = num_roots > num_nodes * a.C ? num_roots : num_nodes * a.C;
  int32_t* state = scratch;
  int32_t* front[2] = {scratch + 8, scratch + 8 + num_points};
  int32_t* cand = scratch + 8 + 2 * num_points;
  int32_t* chunk_cnt = cand + S;
  uint8_t* flags = reinterpret_cast<uint8_t*>(chunk_cnt + 2 * ((S + TREE_THREADS - 1) / TREE_THREADS) + 2);
  tree_init_kernel<<<1, 1, 0, st>>>(state, (int)num_roots, num_roots_d);
  LGR_CHECK_LAUNCH();
  // level 0: the roots themselves
  tree_classify_kernel<true><<<TREE_GRID, TREE_THREADS, 0, st>>>(a, roots, nullptr, state, cand, flags, chunk_cnt);
  LGR_CHECK_LAUNCH();
  tree_scan_kernel<<<1, 1024, 0, st>>>(1, state, chunk_cnt);
  LGR_CHECK_LAUNCH();
  tree_scatter_kernel<<<TREE_GRID, TREE_THREADS, 0, st>>>(1, state, cand, flags, chunk_cnt, out, front[0]);
  LGR_CHECK_LAUNCH();
  tree_advance_kernel<<<1, 1, 0, st>>>(state);
  LGR_CHECK_LAUNCH();
  int cur = 0;
  for (int level = 1; level <= levels; level++) {
    tree_classify_kernel<false><<<TREE_GRID, TREE_THREADS, 0, st>>>(a, nullptr, front[cur], state, cand, flags, chunk_cnt);
    LGR_CHECK_LAUNCH();
    tree_scan_kernel<<<1, 1024, 0, st>>>(a.C, state, chunk_cnt);
    LGR_CHECK_LAUNCH();
    tree_scatter_kernel<<<TREE_GRID, TREE_THREADS, 0, st>>>(a.C, state, cand, flags, chunk_cnt, out, front[cur ^ 1]);
    LGR_CHECK_LAUNCH();
    tree_advance_kernel<<<1, 1, 0, st>>>(state);
    LGR_CHECK_LAUNCH();
    cur ^= 1;
  }
  tree_append_kernel<<<TREE_GRID, TREE_THREADS, 0, st>>>(state, front[cur], out);
  LGR_CHECK_LAUNCH();
  tree_finish_kernel<<<1, 1, 0, st>>>(state, count_out);
  LGR_CHECK_LAUNCH();
  return 0;
}

}  // namespace lgr
