// Fused sparse Adam step for the Gaussians that were visible in the step (SURVEY.md 8(f) row 4), and LoG's whole
// post-backward bookkeeping built on it.
// Reference: LoG/model/sparse_optimizer.py:41-78 (_single_tensor_adam) applied to gathered rows and scattered back
// (:163-196).  One pass: gather moments by index, update, write parameter and moments back in place.  28 bytes of HBM
// traffic per element (32 with amsgrad); the reference runs ~10 elementwise torch kernels per parameter on gathered
// copies plus an index.cpu() synchronisation.
//   sparse_adam_kernel     one key, one thread per (row, float)
//   counter_update_kernel  Counter.update_by_output (LoG/model/counter.py:36-68) for one view: one thread per rendered
//                          row, then one per point_id entry; plain read-modify-writes on unique rows
//   log_step_kernel        LoG.step (level_of_gaussian.py:379-398): every key's Adam update and the scale clamp
//                          (:367-377), one thread per (row, float) across all keys; rows in their own order, or in the
//                          order step_order builds
//   step_order             the flagged rows in ascending Gaussian index for moments held in host memory (read over the
//                          host link, where a row's few bytes per table cost a request each and neighbouring rows share
//                          requests and TLB entries): one byte flag and the row per Gaussian, then lgr_prepare.cu's
//                          order-preserving compaction over the Gaussians -- no sort
//   corrector_step_kernel  Corrector.step (LoG/model/corrector.py:35-62) for one view: one warp, the step count, LoG's
//                          skip before start_step and its learning-rate schedule on the device
#include "lgr_common.cuh"
#include "lgr_prof.cuh"

namespace lgr {

constexpr int ADAM_THREADS = 256;

#ifndef __grid_constant__
#define __grid_constant__      // host compilers of the kernel source: a kernel argument is an ordinary value there
#endif

struct AdamConst {
  float beta1, beta2, one_minus_beta1, one_minus_beta2, bc2_sqrt, neg_step_size, eps;
};

// The update of one element, shared by sparse_adam_kernel and log_step_kernel.
__device__ __forceinline__ void adam_element(float g, float* __restrict__ param, float* __restrict__ exp_avg,
                                             float* __restrict__ exp_avg_sq, float* __restrict__ max_exp_avg_sq,
                                             const AdamConst& a) {
  // explicitly rounded, in the reference's order: m = m*b1 + (1-b1)*g ; v = v*b2 + ((1-b2)*g)*g
  const float m = __fadd_rn(__fmul_rn(*exp_avg, a.beta1), __fmul_rn(a.one_minus_beta1, g));
  const float v = __fadd_rn(__fmul_rn(*exp_avg_sq, a.beta2), __fmul_rn(__fmul_rn(a.one_minus_beta2, g), g));
  *exp_avg = m;
  *exp_avg_sq = v;
  float vv = v;
  if (max_exp_avg_sq) { vv = fmaxf(*max_exp_avg_sq, v); *max_exp_avg_sq = vv; }
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vv), a.bc2_sqrt), a.eps);
  *param = __fadd_rn(*param, __fmul_rn(a.neg_step_size, __fdiv_rn(m, denom)));
}

__global__ void __launch_bounds__(ADAM_THREADS)
sparse_adam_kernel(int64_t total, int C, const int64_t* __restrict__ index, const float* __restrict__ grad,
                   float* __restrict__ param, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                   float* __restrict__ max_exp_avg_sq, AdamConst a) {
  const int64_t t = (int64_t)blockIdx.x * ADAM_THREADS + threadIdx.x;
  if (t >= total) return;
  const int64_t row = t / C;
  const int col = (int)(t - row * C);
  const int64_t dst = index[row] * C + col;
  adam_element(__ldg(grad + t), param + dst, exp_avg + dst, exp_avg_sq + dst, max_exp_avg_sq ? max_exp_avg_sq + dst : nullptr, a);
}

int launch_sparse_adam(int64_t rows, int C, const int64_t* index, const float* grad, float* param, float* exp_avg,
                       float* exp_avg_sq, float* max_exp_avg_sq, float beta1, float beta2, float omb1, float omb2,
                       float bc2_sqrt, float neg_step_size, float eps, cudaStream_t st) {
  const int64_t total = rows * C;
  if (total <= 0) return 0;
  const unsigned blocks = (unsigned)((total + ADAM_THREADS - 1) / ADAM_THREADS);
  const AdamConst a{beta1, beta2, omb1, omb2, bc2_sqrt, neg_step_size, eps};
  sparse_adam_kernel<<<blocks, ADAM_THREADS, 0, st>>>(total, C, index, grad, param, exp_avg, exp_avg_sq, max_exp_avg_sq, a);
  LGR_CHECK_LAUNCH();
  return 0;
}

// ---- LoG's Counter.update_by_output, one view ------------------------------------------------------------------------

// Gaussian of rendered row r: leaves first, then nodes (LoG's torch.cat, counter.py:41-44, level_of_gaussian.py:387-389).
__device__ __forceinline__ int64_t row_gaussian(int64_t r, int64_t num_leaf, const int64_t* __restrict__ leaf,
                                                const int64_t* __restrict__ node) {
  return r < num_leaf ? leaf[r] : node[r - num_leaf];
}

__device__ __forceinline__ int64_t load_int(const void* p, int64_t j, int bytes) {
  return bytes == 8 ? static_cast<const int64_t*>(p)[j] : (int64_t) static_cast<const int32_t*>(p)[j];
}

// torch.norm(grad[:, :2], dim=-1) of one row in fp32: x*x + y*y, each product rounded, then the square root.
__device__ __forceinline__ float norm2_xy(float x, float y) {
  return __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
}

struct CounterArgs {
  lgr_counter c;
  int64_t num_leaf, rows, num_points;
  const int64_t* leaf;
  const int64_t* node;
  const int32_t* radii;
  const float* weight;
  const float* grad;
  int64_t gs0, gs1;
  const void* point_id;
  const void* point_count;
  int id_bytes, count_bytes;
  uint8_t* flag_vis;
};

__global__ void __launch_bounds__(ADAM_THREADS) counter_update_kernel(const __grid_constant__ CounterArgs a) {
  const int64_t t = (int64_t)blockIdx.x * ADAM_THREADS + threadIdx.x;
  if (t < a.rows) {
    const int32_t radius = a.radii[t];
    const bool vis = radius > 0;
    a.flag_vis[t] = vis ? 1 : 0;
    if (!vis) return;
    const int64_t g = row_gaussian(t, a.num_leaf, a.leaf, a.node);
    const float w = a.weight[t];
    a.c.create_steps_d[g] = (int32_t)((uint32_t)a.c.create_steps_d[g] + 1u);
    a.c.visible_count_d[g] = (int16_t)(uint16_t)((uint32_t)(uint16_t)a.c.visible_count_d[g] + 1u);
    const float wm = a.c.weights_max_d[g];
    a.c.weights_max_d[g] = wm != wm ? wm : w != w ? w : fmaxf(wm, w);      // torch.max: NaN propagates
    a.c.weights_sum_d[g] = __fadd_rn(a.c.weights_sum_d[g], w);
    const int16_t r16 = (int16_t)(uint16_t)(uint32_t)radius;
    const int16_t rm = a.c.radii_max_d[g];
    a.c.radii_max_d[g] = r16 > rm ? r16 : rm;
    return;
  }
  const int64_t j = t - a.rows;
  if (j >= a.num_points) return;
  const int64_t p = load_int(a.point_id, j, a.id_bytes);
  const int64_t cnt = load_int(a.point_count, j, a.count_bytes);
  const int64_t g = row_gaussian(p, a.num_leaf, a.leaf, a.node);
  a.c.area_sum_d[g] = (int32_t)((uint32_t)a.c.area_sum_d[g] + (uint32_t)(uint64_t)cnt);
  const float n = norm2_xy(a.grad[p * a.gs0], a.grad[p * a.gs0 + a.gs1]);
  a.c.grad_sum_d[g] = __fadd_rn(a.c.grad_sum_d[g], __fmul_rn(n, (float)cnt));
  const int32_t c32 = (int32_t)(uint32_t)(uint64_t)cnt;
  const int32_t rmm = a.c.radii_max_max_d[g];
  a.c.radii_max_max_d[g] = c32 > rmm ? c32 : rmm;
}

int launch_counter_update(const lgr_counter& c, int64_t num_leaf, int64_t num_node, const int64_t* leaf,
                          const int64_t* node, const int32_t* radii, const float* weight, const float* grad,
                          const int64_t* gs, int64_t num_points, const void* point_id, const void* point_count,
                          int id_bytes, int count_bytes, uint8_t* flag_vis, cudaStream_t st) {
  const int64_t rows = num_leaf + num_node, total = rows + num_points;
  if (total <= 0) return 0;
  const CounterArgs a{c, num_leaf, rows, num_points, leaf, node, radii, weight, grad, gs[0], gs[1], point_id,
                      point_count, id_bytes, count_bytes, flag_vis};
  counter_update_kernel<<<(unsigned)((total + ADAM_THREADS - 1) / ADAM_THREADS), ADAM_THREADS, 0, st>>>(a);
  LGR_CHECK_LAUNCH();
  return 0;
}

// ---- LoG.step: every key's sparse Adam update and the scale clamp, one launch ----------------------------------------

// torch.clamp(v, lo, hi) with tensor bounds: a NaN operand propagates, otherwise min(max(v, lo), hi) (hi where lo > hi).
__device__ __forceinline__ float torch_clamp(float v, float lo, float hi) {
  if (v != v) return v;
  if (lo != lo) return lo;
  if (hi != hi) return hi;
  return fminf(fmaxf(v, lo), hi);
}

__global__ void __launch_bounds__(ADAM_THREADS)
log_step_kernel(const __grid_constant__ lgr_step s, int64_t num_leaf, int64_t total, const int64_t* __restrict__ leaf,
                const int64_t* __restrict__ node, const uint8_t* __restrict__ flag_vis) {
  const int64_t t = (int64_t)blockIdx.x * ADAM_THREADS + threadIdx.x;
  if (t >= total) return;
  const int64_t i = t / s.row_floats;
  const int64_t r = s.order_d ? s.order_d[i] : i;
  if (r < 0 || !flag_vis[r]) return;
  int col = (int)(t - i * s.row_floats), k = 0;
  while (k + 1 < s.num_keys && col >= s.keys[k + 1].prefix) k++;
  const lgr_step_key& key = s.keys[k];
  col -= key.prefix;
  const int64_t g = row_gaussian(r, num_leaf, leaf, node);
  const int64_t dst = g * key.row_floats + col;
  if (key.grad_d) {
    const AdamConst a{s.beta1, s.beta2, s.one_minus_beta1, s.one_minus_beta2, key.bc2_sqrt, key.neg_step_size, s.eps};
    adam_element(__ldg(key.grad_d + r * key.row_floats + col), key.param_d + dst, key.exp_avg_d + dst,
                 key.exp_avg_sq_d + dst, key.max_exp_avg_sq_d ? key.max_exp_avg_sq_d + dst : nullptr, a);
  }
  if (key.clamp)
    key.param_d[dst] = torch_clamp(key.param_d[dst], logf(s.radius3d_min_d[g]), logf(s.radius3d_max_d[g]));
}

int launch_log_step(const lgr_step& s, int64_t num_leaf, int64_t num_node, const int64_t* leaf, const int64_t* node,
                    const uint8_t* flag_vis, cudaStream_t st) {
  const int64_t total = (num_leaf + num_node) * s.row_floats;
  if (total <= 0) return 0;
  log_step_kernel<<<(unsigned)((total + ADAM_THREADS - 1) / ADAM_THREADS), ADAM_THREADS, 0, st>>>(s, num_leaf, total, leaf,
                                                                                                 node, flag_vis);
  LGR_CHECK_LAUNCH();
  return 0;
}

// ---- the ordered pass: flagged rows in ascending Gaussian index ------------------------------------------------------

constexpr int ORDER_THREADS = COMPACT_CHUNK;
#ifndef LGR_TREE_GRID
#define LGR_TREE_GRID 528               // 4 CTAs per SM on the 132 SMs of an H100 SXM; grid-stride loops cover any size
#endif

int launch_compact_scan(int64_t, int32_t*, int64_t*, int64_t*, cudaStream_t);
int launch_compact_scatter(int64_t, const uint8_t*, const int32_t*, const int32_t*, int64_t*, int64_t*, cudaStream_t);

// bits[g] = 1 and row_of[g] = r for every flagged row r (bits zeroed before)
__global__ void __launch_bounds__(ORDER_THREADS)
step_mark_kernel(int64_t rows, int64_t num_leaf, const int64_t* __restrict__ leaf, const int64_t* __restrict__ node,
                 const uint8_t* __restrict__ flag_vis, int64_t n, uint8_t* __restrict__ bits, int32_t* __restrict__ row_of) {
  for (int64_t r = (int64_t)blockIdx.x * ORDER_THREADS + threadIdx.x; r < rows; r += (int64_t)gridDim.x * ORDER_THREADS) {
    if (!flag_vis[r]) continue;
    const int64_t g = row_gaussian(r, num_leaf, leaf, node);
    if ((uint64_t)g >= (uint64_t)n) continue;
    bits[g] = 1;
    row_of[g] = (int32_t)r;
  }
}

// the flagged Gaussians of each chunk, as the (A, B) pairs lgr_prepare.cu's scan takes (B empty)
__global__ void __launch_bounds__(ORDER_THREADS)
step_count_kernel(int64_t n, const uint8_t* __restrict__ bits, int32_t* __restrict__ chunk_cnt) {
  const int64_t nchunks = (n + ORDER_THREADS - 1) / ORDER_THREADS;
  for (int64_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    const int64_t g = chunk * ORDER_THREADS + threadIdx.x;
    const int c = __syncthreads_count(g < n && bits[g]);
    if (threadIdx.x == 0) { chunk_cnt[2 * chunk] = c; chunk_cnt[2 * chunk + 1] = 0; }
  }
}

// scratch layout (int32 units): count [2, one int64] | chunk counts [2 ceil(n/256) + 2] | row_of [n] | bits [n bytes]
int launch_step_order(int64_t n, int64_t num_leaf, int64_t num_node, const int64_t* leaf, const int64_t* node,
                      const uint8_t* flag_vis, int32_t* scratch, int64_t* order, cudaStream_t st) {
  const int64_t rows = num_leaf + num_node;
  if (rows == 0) return 0;
  cudaError_t e = cudaMemsetAsync(order, 0xff, sizeof(int64_t) * (size_t)rows, st);      // -1 past the count
  if (e != cudaSuccess || n == 0) return (int)e;
  int64_t* count = reinterpret_cast<int64_t*>(scratch);
  int32_t* chunk_cnt = scratch + 2;
  int32_t* row_of = chunk_cnt + 2 * ((n + ORDER_THREADS - 1) / ORDER_THREADS) + 2;
  uint8_t* bits = reinterpret_cast<uint8_t*>(row_of + n);
  e = cudaMemsetAsync(bits, 0, (size_t)n, st);
  if (e != cudaSuccess) return (int)e;
  step_mark_kernel<<<LGR_TREE_GRID, ORDER_THREADS, 0, st>>>(rows, num_leaf, leaf, node, flag_vis, n, bits, row_of);
  LGR_CHECK_LAUNCH();
  step_count_kernel<<<LGR_TREE_GRID, ORDER_THREADS, 0, st>>>(n, bits, chunk_cnt);
  LGR_CHECK_LAUNCH();
  const int rc = launch_compact_scan(n, chunk_cnt, count, nullptr, st);
  if (rc) return rc;
  return launch_compact_scatter(n, bits, chunk_cnt, row_of, order, nullptr, st);
}

// ---- Corrector.step: one row of the (V, 3) view-correction table ----------------------------------------------------

// fp64 products and sums rounded one by one, as numpy's (no contraction into a fused multiply-add).
__device__ __forceinline__ double dmul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__device__ __forceinline__ double dadd_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

// One warp.  steps[i] += 1 (int32 wrap); s = steps[i] - start_step; s < 0 returns (the gradient row keeps accumulating,
// as in LoG).  Otherwise lanes 0..2 update one column each.
//   lr = exp(log lr_init (1 - t) + log lr_final t), t = clip(s / 100, 0, 1): numpy's float64 operations in numpy's
//     order, each rounded; the two logs come from numpy on the host.  exp is the CUDA math library's (max 1 ulp in
//     fp64), which may differ from numpy's in the last bit of the double; lr enters as (float)lr, where that shows only
//     if the double lies within an ulp of a float rounding boundary.
//   The bias corrections as LoG's _single_tensor_adam computes them with a tensor step, in float32 tensor operations:
//     1 - 0.9^s, sqrt(1 - 0.999^s) and step_size = (1 / bc1) * (float)lr (Tensor.__rtruediv__ is reciprocal() * lr).
//   The moments as torch's CUDA kernels compute LoG's in-place ops, the rounding LoG gets when it trains on the GPU:
//     exp_avg.mul_(b1).add_(g, alpha=1-b1) is fma(1-b1, g, m*b1) (AddFunctor a + alpha*b, contracted), and
//     exp_avg_sq.mul_(b2).addcmul_(g, g, value=1-b2) is fma(1-b2, g*g, v*b2) (a + alpha*(b*c), contracted).  torch's
//     CPU addcmul_ rounds the second as fma((1-b2)*g, g, v*b2) instead; adam_element rounds every product separately.
//   AMSGrad maximum (NaN propagates, as torch.max), denominator and update in torch's order; then grad[i] = 0.
__global__ void __launch_bounds__(32)
corrector_step_kernel(int64_t index, int32_t start_step, double log_lr_init, double log_lr_final, int32_t* __restrict__ steps,
                      float* __restrict__ param, float* __restrict__ grad, float* __restrict__ exp_avg,
                      float* __restrict__ exp_avg_sq, float* __restrict__ max_exp_avg_sq) {
  const int lane = threadIdx.x;
  const int32_t count = (int32_t)((uint32_t)steps[index] + 1u);
  __syncwarp();
  if (lane == 0) steps[index] = count;
  const int32_t s = (int32_t)((uint32_t)count - (uint32_t)start_step);
  if (s < 0 || lane >= 3) return;
  const double t = fmin(fmax((double)s / 100.0, 0.0), 1.0);
  const double lr = exp(dadd_rn(dmul_rn(log_lr_init, 1.0 - t), dmul_rn(log_lr_final, t)));
  const float sf = (float)s;
  const float bc1 = __fsub_rn(1.f, powf(0.9f, sf)), bc2 = __fsub_rn(1.f, powf(0.999f, sf));
  const float step_size = __fmul_rn(__fdiv_rn(1.f, bc1), (float)lr);
  const float omb1 = (float)(1.0 - 0.9), omb2 = (float)(1.0 - 0.999);
  const int64_t e = index * 3 + lane;
  const float g = grad[e];
  const float m = __fmaf_rn(omb1, g, __fmul_rn(exp_avg[e], 0.9f));
  const float v = __fmaf_rn(omb2, __fmul_rn(g, g), __fmul_rn(exp_avg_sq[e], 0.999f));
  exp_avg[e] = m;
  exp_avg_sq[e] = v;
  float vv = v;
  if (max_exp_avg_sq) {
    const float vm = max_exp_avg_sq[e];
    vv = vm != vm ? vm : v != v ? v : fmaxf(vm, v);      // torch.max: NaN propagates
    max_exp_avg_sq[e] = vv;
  }
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vv), __fsqrt_rn(bc2)), 1e-15f);
  param[e] = __fadd_rn(param[e], __fmul_rn(-step_size, __fdiv_rn(m, denom)));
  grad[e] = 0.f;
}

int launch_corrector_step(int64_t index, int32_t start_step, double log_lr_init, double log_lr_final, int32_t* steps,
                          float* param, float* grad, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq,
                          cudaStream_t st) {
  corrector_step_kernel<<<1, 32, 0, st>>>(index, start_step, log_lr_init, log_lr_final, steps, param, grad, exp_avg,
                                          exp_avg_sq, max_exp_avg_sq);
  LGR_CHECK_LAUNCH();
  return 0;
}

}  // namespace lgr
