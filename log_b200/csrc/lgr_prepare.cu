// LoG.prepare (LoG/model/level_of_gaussian.py:223-256, Gaussian.prepare at :90-98) on the device: the per-view selection
// of the Gaussians a training step renders, with no host synchronisation between its stages.
//
//   cull     one thread per root (tree mode) or per point (base stage): LoG's frustum test (_visible_flag_by_camera, :40-53)
//            in fp32, the flag byte, and a stable compaction of the in-range ids in id order
//   (the caller renders the in-range roots with the ordinary forward: gather list = the compacted roots, -1 past the count)
//   merge    one thread per rendered root: root_flag[j] = 0 where point_weight <= 1e-8 (render_to_check, :233-241), the
//            surviving roots compacted in root order: the walk's first frontier
//   walk     lgr_tree.cu, seeded from the survivor count on the device
//   split    one thread per walk entry: LoG's leaf / node rule (:244-251), two order-preserving lists
//
// Every compaction is the pattern of lgr_tree.cu: a fixed grid of grid-stride loops over a count that may live on the
// device, per-chunk counts, a one-CTA exclusive scan (cta_exclusive_scan), then chunk prefix + ballot rank
// (cta_ballot_rank).  The counts land in the (int64) result vector the host reads once.
#include "lgr_common.cuh"

namespace lgr {

constexpr int PREP_THREADS = COMPACT_CHUNK;
#ifndef LGR_TREE_GRID
#define LGR_TREE_GRID 528               // 4 CTAs per SM on the 132 SMs of an H100 SXM; grid-stride loops cover any size
#endif
constexpr int PREP_GRID = LGR_TREE_GRID;

enum PrepMode { CULL_ROOTS = 0, CULL_POINTS = 1, MERGE = 2, SPLIT = 3 };

struct PrepArgs {
  const float* xyz;            // (P,3)
  const float* M;              // (4,4) full_proj_transform, row-vector convention: [x y z 1] @ M
  float lo, hi;                // -1 - padding, 1 + padding, rounded to fp32 as torch compares them
  const int32_t* root_index;   // (R)
  int64_t num_points;
  const int32_t* node_index;   // (P)
  const int8_t* depth;         // (P)
  int opt_all_levels, current_depth;
  uint8_t* flag;               // (R) root_flag or (P) flag
  const int64_t* in_range;     // (R) the rendered roots (merge)
  const float* point_weight;   // (R) their point_weight (merge)
  const int64_t* index_all;    // the walk's output (split)
  int64_t* result;             // LGR_PREPARE_RESULTS
};

// xyz1 @ M, pw = 1 / (w + 1e-7), p = xyz * pw, then LoG's six comparisons.  Explicitly rounded intrinsics, so the
// compiler neither contracts nor reorders; the sums run x, y, z, then the constant row.  1.0f / t is IEEE division (no
// fast-math), as torch's reciprocal.
__device__ __forceinline__ bool log_in_frustum(const PrepArgs& a, int64_t id) {
  const float x = a.xyz[3 * id], y = a.xyz[3 * id + 1], z = a.xyz[3 * id + 2];
  float h[4];
#pragma unroll
  for (int k = 0; k < 4; k++)
    h[k] = __fadd_rn(__fmaf_rn(z, a.M[8 + k], __fmaf_rn(y, a.M[4 + k], __fmul_rn(x, a.M[k]))), a.M[12 + k]);
  const float pw = 1.0f / __fadd_rn(h[3], 1e-7f);
  const float px = __fmul_rn(h[0], pw), py = __fmul_rn(h[1], pw), pz = __fmul_rn(h[2], pw);
  return (pz > 0.f) & (pz < 1.f) & (px > a.lo) & (px < a.hi) & (py > a.lo) & (py < a.hi);
}

// bits[slot]: bit 0 = list A, bit 1 = list B; cand[slot] = the id the slot contributes; two counts per chunk
template <int MODE>
__global__ void __launch_bounds__(PREP_THREADS)
prep_classify_kernel(PrepArgs a, int64_t n_host, const int64_t* __restrict__ n_d, int64_t* __restrict__ cand,
                     uint8_t* __restrict__ bits, int32_t* __restrict__ chunk_cnt) {
  const int64_t n = n_d ? *n_d : n_host;
  const int64_t nchunks = (n + PREP_THREADS - 1) / PREP_THREADS;
  for (int64_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    const int64_t slot = chunk * PREP_THREADS + threadIdx.x;
    int f = 0;
    if (slot < n) {
      int64_t id = slot;
      if (MODE == CULL_ROOTS) {
        // LoG tests xyz[root_index][j] but renders the table rows root_index[flag]: one Gaussian only when root_index[j] == j
        const int64_t r = a.root_index[slot];
        const bool ok = r == slot;
        if (!ok) a.result[LGR_PREPARE_STATUS] = LGR_PREPARE_ROOT_ORDER;      // every writer stores the same value
        f = (ok && log_in_frustum(a, r)) ? 1 : 0;
        a.flag[slot] = (uint8_t)f;
      } else if (MODE == CULL_POINTS) {
        f = log_in_frustum(a, slot) ? 1 : 0;
        a.flag[slot] = (uint8_t)f;
      } else if (MODE == MERGE) {
        id = a.in_range[slot];
        f = a.point_weight[slot] > 1e-8f ? 1 : 0;
        if (!f) a.flag[id] = 0;
      } else {
        id = a.index_all[slot];
        const int d = a.depth[id];
        const bool leaf = a.opt_all_levels ? (a.node_index[id] == -1 && d > 0) : d == a.current_depth;
        f = leaf ? 1 : 2;
      }
      cand[slot] = id;
      bits[slot] = (uint8_t)f;
    }
    const int na = __syncthreads_count(f & 1), nb = __syncthreads_count(f & 2);
    if (threadIdx.x == 0) { chunk_cnt[2 * chunk] = na; chunk_cnt[2 * chunk + 1] = nb; }
  }
}

// exclusive scan of the (A, B) chunk counts in place; the totals go to total_a / total_b (either may be null)
__global__ void __launch_bounds__(1024)
prep_scan_kernel(int64_t n_host, const int64_t* __restrict__ n_d, int32_t* __restrict__ chunk_cnt, int64_t* __restrict__ total_a,
                 int64_t* __restrict__ total_b) {
  const int64_t n = n_d ? *n_d : n_host;
  const ScanTotals<2> t = cta_exclusive_scan<1024, 2>((int)((n + PREP_THREADS - 1) / PREP_THREADS),
                                                      [&](int b, int k) { return chunk_cnt[2 * b + k]; },
                                                      [&](int b, int k, int pre) { chunk_cnt[2 * b + k] = pre; });
  if (threadIdx.x == 0) {
    if (total_a) *total_a = t.v[0];
    if (total_b) *total_b = t.v[1];
  }
}

// stable compaction: A-slots to out_a, B-slots to out_b, each in slot order; a slot contributes cand[slot], or the slot
// itself when cand is null.  pad_a: out_a[total_a .. n) = -1 (the gather list of the visibility render, whose rows past
// the count are empty)
template <class Cand>
__global__ void __launch_bounds__(PREP_THREADS)
prep_scatter_kernel(int64_t n_host, const int64_t* __restrict__ n_d, const Cand* __restrict__ cand,
                    const uint8_t* __restrict__ bits, const int32_t* __restrict__ chunk_pre, int64_t* __restrict__ out_a,
                    int64_t* __restrict__ out_b, const int64_t* __restrict__ total_a, int pad_a) {
  __shared__ __align__(16) int wa[PREP_THREADS / 32];
  __shared__ __align__(16) int wb[PREP_THREADS / 32];
  const int64_t n = n_d ? *n_d : n_host;
  const int64_t nchunks = (n + PREP_THREADS - 1) / PREP_THREADS;
  for (int64_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    const int64_t slot = chunk * PREP_THREADS + threadIdx.x;
    const int f = slot < n ? bits[slot] : 0;
    const int ra = cta_ballot_rank<PREP_THREADS>(f & 1, wa).rank, rb = cta_ballot_rank<PREP_THREADS>(f & 2, wb).rank;
    if (f & 1) out_a[chunk_pre[2 * chunk] + ra] = cand ? (int64_t)cand[slot] : slot;
    if (f & 2) out_b[chunk_pre[2 * chunk + 1] + rb] = cand ? (int64_t)cand[slot] : slot;
  }
  if (pad_a) {
    const int64_t t = *total_a;
    for (int64_t i = t + (int64_t)blockIdx.x * PREP_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * PREP_THREADS) out_a[i] = -1;
  }
}

// the visibility render's instance count and overflow flags, next to the counts: one read for the host
__global__ void prep_finish_kernel(const int32_t* __restrict__ meta, int64_t* __restrict__ result) {
  result[LGR_PREPARE_INSTANCES] = meta ? (int64_t)(uint32_t)meta[0] : 0;
  result[LGR_PREPARE_OVERFLOW] = meta ? (int64_t)meta[6] : 0;
}

struct PrepScratch {
  int64_t* cand;
  uint8_t* bits;
  int32_t* chunk_cnt;
  int32_t* walk;
};

// scratch layout (int32 units): cand [2 P] | chunk counts [2 ceil(P/256) + 2] | bits [P bytes] | walk scratch
static PrepScratch prep_scratch(int32_t* scratch, int64_t p) {
  PrepScratch s;
  s.cand = reinterpret_cast<int64_t*>(scratch);
  s.chunk_cnt = scratch + 2 * p;
  s.bits = reinterpret_cast<uint8_t*>(s.chunk_cnt + 2 * ((p + PREP_THREADS - 1) / PREP_THREADS) + 2);
  s.walk = reinterpret_cast<int32_t*>(s.bits) + (p + 3) / 4;
  return s;
}

template <int MODE>
static int prep_compact(const PrepArgs& a, const PrepScratch& s, int64_t n_host, const int64_t* n_d, int64_t* out_a,
                        int64_t* out_b, int64_t* total_a, int64_t* total_b, bool pad_a, cudaStream_t st) {
  prep_classify_kernel<MODE><<<PREP_GRID, PREP_THREADS, 0, st>>>(a, n_host, n_d, s.cand, s.bits, s.chunk_cnt);
  LGR_CHECK_LAUNCH();
  prep_scan_kernel<<<1, 1024, 0, st>>>(n_host, n_d, s.chunk_cnt, total_a, total_b);
  LGR_CHECK_LAUNCH();
  prep_scatter_kernel<int64_t><<<PREP_GRID, PREP_THREADS, 0, st>>>(n_host, n_d, s.cand, s.bits, s.chunk_cnt, out_a, out_b,
                                                                 total_a, pad_a ? 1 : 0);
  LGR_CHECK_LAUNCH();
  return 0;
}

// The scan and the scatter of a compaction whose classify pass lives in another file (lgr_densify.cu, lgr_optim.cu): bits
// and chunk counts as prep_classify_kernel writes them, chunks of COMPACT_CHUNK slots, and as the output cand[slot], or
// the slot ids when cand is null.
int launch_compact_scan(int64_t n, int32_t* chunk_cnt, int64_t* total_a, int64_t* total_b, cudaStream_t st) {
  prep_scan_kernel<<<1, 1024, 0, st>>>(n, nullptr, chunk_cnt, total_a, total_b);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_compact_scatter(int64_t n, const uint8_t* bits, const int32_t* chunk_pre, const int32_t* cand, int64_t* out_a,
                           int64_t* out_b, cudaStream_t st) {
  prep_scatter_kernel<int32_t><<<PREP_GRID, PREP_THREADS, 0, st>>>(n, nullptr, cand, bits, chunk_pre, out_a, out_b, nullptr, 0);
  LGR_CHECK_LAUNCH();
  return 0;
}

static PrepArgs prep_args(const lgr_prepare& p) {
  PrepArgs a;
  a.xyz = p.xyz_d; a.M = p.full_proj_d; a.lo = p.bound_lo; a.hi = p.bound_hi;
  a.root_index = p.root_index_d; a.num_points = p.num_points;
  a.node_index = p.node_index_d; a.depth = p.depth_d;
  a.opt_all_levels = p.opt_all_levels; a.current_depth = p.current_depth;
  a.flag = p.flag_d; a.in_range = p.in_range_d; a.point_weight = nullptr; a.index_all = p.index_all_d;
  a.result = p.result_d;
  return a;
}

int launch_prepare_cull(const lgr_prepare& p, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(p.result_d, 0, LGR_PREPARE_RESULTS * sizeof(int64_t), st);
  if (e != cudaSuccess) return (int)e;
  const PrepArgs a = prep_args(p);
  const PrepScratch s = prep_scratch(p.scratch_d, p.num_points);
  if (p.num_roots > 0)
    return prep_compact<CULL_ROOTS>(a, s, p.num_roots, nullptr, p.in_range_d, nullptr, p.result_d + LGR_PREPARE_IN_RANGE, nullptr,
                                    true, st);
  return prep_compact<CULL_POINTS>(a, s, p.num_points, nullptr, p.in_range_d, nullptr, p.result_d + LGR_PREPARE_IN_RANGE, nullptr,
                                   false, st);
}

int launch_tree_traverse(const TreeArgs&, int64_t, int64_t, const int64_t*, int64_t, const int64_t*, int, int32_t*, int64_t*, int64_t*,
                         cudaStream_t);

int launch_prepare_select(const lgr_prepare& p, const TreeArgs& t, int64_t num_nodes, int levels, const float* point_weight,
                          const int32_t* meta, cudaStream_t st) {
  PrepArgs a = prep_args(p);
  a.point_weight = point_weight;
  const PrepScratch s = prep_scratch(p.scratch_d, p.num_points);
  int64_t* res = p.result_d;
  int rc = prep_compact<MERGE>(a, s, 0, res + LGR_PREPARE_IN_RANGE, p.roots_d, nullptr, res + LGR_PREPARE_ROOTS, nullptr, false, st);
  if (rc) return rc;
  rc = launch_tree_traverse(t, p.num_points, num_nodes, p.roots_d, p.num_roots, res + LGR_PREPARE_ROOTS, levels, s.walk,
                            p.index_all_d, res + LGR_PREPARE_WALK, st);
  if (rc) return rc;
  rc = prep_compact<SPLIT>(a, s, 0, res + LGR_PREPARE_WALK, p.leaf_d, p.node_d, res + LGR_PREPARE_LEAVES, res + LGR_PREPARE_NODES,
                           false, st);
  if (rc) return rc;
  prep_finish_kernel<<<1, 1, 0, st>>>(meta, res);
  LGR_CHECK_LAUNCH();
  return 0;
}

}  // namespace lgr
