// LoG's depth-supervision loss and its gradient (NaiveRendererAndLoss.append_depth_loss, LoG/render/renderer.py:268-292,
// with MiDaS's ScaleAndShiftInvariantLoss(alpha=0.5, scales=1), LoG/render/loss.py:47-117).  LoG cuts 64 random 64x64
// patches in a Python loop (each slice bound an item()), fits a scale and shift per patch with det.nonzero(), and its
// backward sums 64 zero-filled full-size gradients.  Here, with the corners as device data and no host round trip:
//   depth_patch_fwd_kernel   one CTA per patch: stage it, the five moments about a local centre in fp64, the 2x2 solve,
//                            then a second pass for the data term, the regulariser and the masked count
//   depth_loss_reduce_kernel one thread: the 64 patch sums in patch order -> loss (float) and 1/M for the backward
//   depth_patch_bwd_kernel   one CTA per patch: dL/ds and dL/dt of the regulariser by a block reduction, then dL/dd per
//                            pixel of the patch into a (64, 64*64) scratch
//   depth_grad_map_kernel    the dense (H, W) gradient: each pixel sums the patches that cover it in patch order, zero
//                            where none does (no float atomics: loss and gradient repeat bit for bit)
//   depth_vis_minmax_kernel, depth_vis_kernel   LoG's visualisation (q - min q) / (max q - min q) over the masked pixels,
//                            q = 1/(d + 1e-5) with IEEE division in fp32, bit for bit what torch computes
// Every map is read through 2-D element strides, so the depth and accmap planes of the (6, H, W) render are not copied.
//
// Notation, per patch: m the mask (accmap > 0.5), q = 1/(d + 1e-5), g the ground truth, c the q of the patch's first
// masked pixel, u = q - c.  The fit ssi = s q + t = s u + t' (t = t' - s c) solves the normal equations of
// sum m (s u + t' - g)^2; r = ssi - g on masked pixels.
#include "lgr_common.cuh"
#include <math.h>

namespace lgr {

constexpr int DP = LGR_DEPTH_PATCH;              // patch edge
constexpr int DN = LGR_DEPTH_PATCHES;            // patches per call
constexpr int DPIX = DP * DP;
constexpr int D_THREADS = 256;
constexpr int D_PER = DPIX / D_THREADS;          // pixels per thread
constexpr int D_WARPS = D_THREADS / 32;
constexpr int D_STAT = LGR_DEPTH_STAT_DOUBLES_PER_PATCH;
// dynamic shared memory of the patch kernels: u (double), g (float), the mask (bits)
constexpr int D_SMEM = DPIX * (int)sizeof(double) + DPIX * (int)sizeof(float) + DPIX / 8;
// per-patch record in the stats buffer: the fit, the moments the backward needs, and the patch's loss partial
enum { ST_S = 0, ST_T, ST_C, ST_N, ST_SU, ST_SUU, ST_DET, ST_PART };

struct DepthArgs {
  int H, W, Hd, Wd;
  int64_t sp[2], sa[2], sg[2];     // element strides (row, column) of pred, accmap, gt
};

__device__ __forceinline__ double depth_q(float d) { return 1.0 / ((double)d + 1e-5); }
__device__ __forceinline__ float depth_vis_q(float d) { return 1.0f / (d + 1e-5f); }     // torch's reciprocal in fp32
__device__ __forceinline__ bool depth_bit(const unsigned* m, int i) { return (m[i >> 5] >> (i & 31)) & 1u; }
__device__ __forceinline__ double depth_sign(double x) { return (double)((x > 0.0) - (x < 0.0)); }
// min / max that propagate NaN, as torch's reductions do
__device__ __forceinline__ float depth_min(float a, float b) { return (a < b || a != a) ? a : b; }
__device__ __forceinline__ float depth_max(float a, float b) { return (a > b || a != a) ? a : b; }

// Block-wide sums of N doubles in a fixed order (warp tree, then the warps in index order), returned to every thread.
template <int N>
__device__ __forceinline__ void depth_block_sum(double (&v)[N], double (*red)[D_WARPS]) {
#pragma unroll
  for (int n = 0; n < N; n++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[n] += __shfl_down_sync(0xffffffffu, v[n], o);
    if ((threadIdx.x & 31) == 0) red[n][threadIdx.x >> 5] = v[n];
  }
  __syncthreads();
#pragma unroll
  for (int n = 0; n < N; n++) {
    double s = 0.0;
    for (int w = 0; w < D_WARPS; w++) s += red[n][w];
    v[n] = s;
  }
  __syncthreads();      // red is reused by the next call
}

// The patch's corner, or false when the 64x64 patch does not lie inside the ground truth (nothing is read then).
__device__ __forceinline__ bool depth_corner(const DepthArgs& a, const int64_t* rows, const int64_t* cols, int k, int& r0,
                                             int& c0) {
  const int64_t r = rows[k], c = cols[k];
  if (r < 0 || c < 0 || r > a.Hd - DP || c > a.Wd - DP) return false;
  r0 = (int)r;
  c0 = (int)c;
  return true;
}

// Stage one patch: su <- u = q - c (0 where unmasked), sg <- g, sm <- the mask as bits.  Returns c (0 when the patch has
// no masked pixel).  Centring makes the moments' determinant exactly 0 when every masked q is equal.  u is kept in
// double: the regulariser's sign(r_i - r_j) flips wherever r is rounded more coarsely than the neighbours differ.
__device__ double depth_stage(const DepthArgs& a, const float* __restrict__ pred, const float* __restrict__ acc,
                              const float* __restrict__ gt, int r0, int c0, double* su, float* sg, unsigned* sm) {
#pragma unroll 4
  for (int j = 0; j < D_PER; j++) {
    const int i = j * D_THREADS + threadIdx.x, y = r0 + i / DP, x = c0 + i % DP;
    const bool in = acc[y * a.sa[0] + x * a.sa[1]] > 0.5f;
    su[i] = pred[y * a.sp[0] + x * a.sp[1]];
    sg[i] = gt[y * a.sg[0] + x * a.sg[1]];
    const unsigned bits = __ballot_sync(0xffffffffu, in);
    if ((threadIdx.x & 31) == 0) sm[i >> 5] = bits;
  }
  __syncthreads();
  int first = -1;
  for (int w = 0; w < DPIX / 32; w++)
    if (sm[w]) {
      first = w * 32 + __ffs((int)sm[w]) - 1;
      break;
    }
  const double c = first < 0 ? 0.0 : depth_q((float)su[first]);
  __syncthreads();      // every thread has read su[first]
#pragma unroll 4
  for (int j = 0; j < D_PER; j++) {
    const int i = j * D_THREADS + threadIdx.x;
    su[i] = depth_bit(sm, i) ? depth_q((float)su[i]) - c : 0.0;
  }
  __syncthreads();
  return c;
}

// r = s u + t' - g, with one rounding order everywhere it is evaluated (the regulariser compares neighbours' r)
__device__ __forceinline__ double depth_res(double s, double t, const double* su, const float* sg, int i) {
  return fma(s, su[i], t) - (double)sg[i];
}

__global__ void __launch_bounds__(D_THREADS)
depth_patch_fwd_kernel(const DepthArgs a, const float* __restrict__ pred, const float* __restrict__ acc,
                       const float* __restrict__ gt, const int64_t* __restrict__ rows, const int64_t* __restrict__ cols,
                       double* __restrict__ stats) {
  extern __shared__ double depth_smem[];
  double* su = depth_smem;
  float* sg = reinterpret_cast<float*>(su + DPIX);
  unsigned* sm = reinterpret_cast<unsigned*>(sg + DPIX);
  __shared__ double red[5][D_WARPS];
  double* st = stats + (int64_t)blockIdx.x * D_STAT;
  int r0, c0;
  if (!depth_corner(a, rows, cols, blockIdx.x, r0, c0)) {
    if (threadIdx.x < D_STAT) st[threadIdx.x] = threadIdx.x == ST_PART ? (double)NAN : 0.0;
    return;
  }
  const double c = depth_stage(a, pred, acc, gt, r0, c0, su, sg, sm);
  double mo[5] = {0.0, 0.0, 0.0, 0.0, 0.0};      // n, sum u, sum u^2, sum g, sum u g over the masked pixels
  for (int j = 0; j < D_PER; j++) {
    const int i = j * D_THREADS + threadIdx.x;
    if (!depth_bit(sm, i)) continue;
    const double u = su[i], g = sg[i];
    mo[0] += 1.0; mo[1] += u; mo[2] += u * u; mo[3] += g; mo[4] += u * g;
  }
  depth_block_sum<5>(mo, red);
  const double n = mo[0], Su = mo[1], Suu = mo[2], Sg = mo[3], Sug = mo[4];
  const double det = n * Suu - Su * Su;
  double s = 0.0, t = 0.0;      // LoG's s = t = 0 where det == 0 (no, one, or only equal masked q)
  if (det != 0.0) {
    s = (n * Sug - Su * Sg) / det;
    t = (Suu * Sg - Su * Sug) / det;
  }
  double e[2] = {0.0, 0.0};      // sum m r^2, sum over masked neighbour pairs |r_j - r_i|
  for (int j = 0; j < D_PER; j++) {
    const int i = j * D_THREADS + threadIdx.x, x = i % DP, y = i / DP;
    if (!depth_bit(sm, i)) continue;
    const double r = depth_res(s, t, su, sg, i);
    e[0] += r * r;
    if (x + 1 < DP && depth_bit(sm, i + 1)) e[1] += fabs(depth_res(s, t, su, sg, i + 1) - r);
    if (y + 1 < DP && depth_bit(sm, i + DP)) e[1] += fabs(depth_res(s, t, su, sg, i + DP) - r);
  }
  depth_block_sum<2>(e, red);
  if (threadIdx.x == 0) {
    st[ST_S] = s; st[ST_T] = t; st[ST_C] = c; st[ST_N] = n; st[ST_SU] = Su; st[ST_SUU] = Suu; st[ST_DET] = det;
    st[ST_PART] = e[0] + 0.5 * e[1];
  }
}

// loss = sum_k part_k / M, M = sum_k n_k; stats[DN * D_STAT] = 1/M for the backward.  M = 0 (empty mask) gives NaN, as
// LoG's 0/0.
__global__ void depth_loss_reduce_kernel(double* __restrict__ stats, float* __restrict__ loss) {
  if (threadIdx.x != 0) return;
  double sum = 0.0, M = 0.0;
  for (int k = 0; k < DN; k++) {
    sum += stats[k * D_STAT + ST_PART];
    M += stats[k * D_STAT + ST_N];
  }
  stats[DN * D_STAT] = 1.0 / M;
  *loss = (float)(sum / M);
}

// Per patch, dL_k/dd (without the common factor dL/dloss / M) into scratch[k][64*64]:
//   dL_k/dq_i = e_i s + m_i (-l0 (r_i + u_i s) - l1 s),   e_i = 2 r_i + 0.5 sum_{masked neighbours j} sign(r_i - r_j)
// with (l0, l1) = A^-1 (dL/ds, dL/dt) through the centred normal matrix A = [[Suu, Su], [Su, n]], and dq/dd = -q^2.
// Only the regulariser enters dL/ds, dL/dt: the data term's share is zero at the least-squares fit.
__global__ void __launch_bounds__(D_THREADS)
depth_patch_bwd_kernel(const DepthArgs a, const float* __restrict__ pred, const float* __restrict__ acc,
                       const float* __restrict__ gt, const int64_t* __restrict__ rows, const int64_t* __restrict__ cols,
                       const double* __restrict__ stats, float* __restrict__ scratch) {
  extern __shared__ double depth_smem[];
  double* su = depth_smem;
  float* sg = reinterpret_cast<float*>(su + DPIX);
  unsigned* sm = reinterpret_cast<unsigned*>(sg + DPIX);
  __shared__ double red[2][D_WARPS];
  float* out = scratch + (int64_t)blockIdx.x * DPIX;
  int r0, c0;
  if (!depth_corner(a, rows, cols, blockIdx.x, r0, c0)) {
    for (int i = threadIdx.x; i < DPIX; i += D_THREADS) out[i] = NAN;
    return;
  }
  const double c = depth_stage(a, pred, acc, gt, r0, c0, su, sg, sm);
  const double* st = stats + (int64_t)blockIdx.x * D_STAT;
  const double s = st[ST_S], t = st[ST_T], n = st[ST_N], Su = st[ST_SU], Suu = st[ST_SUU], det = st[ST_DET];
  double er[D_PER];      // the regulariser's dL/dr per pixel
  double v[2] = {0.0, 0.0};
#pragma unroll
  for (int j = 0; j < D_PER; j++) {
    const int i = j * D_THREADS + threadIdx.x, x = i % DP, y = i / DP;
    er[j] = 0.0;
    if (!depth_bit(sm, i)) continue;
    const double r = depth_res(s, t, su, sg, i);
    if (x > 0 && depth_bit(sm, i - 1)) er[j] += depth_sign(r - depth_res(s, t, su, sg, i - 1));
    if (x + 1 < DP && depth_bit(sm, i + 1)) er[j] += depth_sign(r - depth_res(s, t, su, sg, i + 1));
    if (y > 0 && depth_bit(sm, i - DP)) er[j] += depth_sign(r - depth_res(s, t, su, sg, i - DP));
    if (y + 1 < DP && depth_bit(sm, i + DP)) er[j] += depth_sign(r - depth_res(s, t, su, sg, i + DP));
    er[j] *= 0.5;
    v[0] += er[j] * su[i];
    v[1] += er[j];
  }
  depth_block_sum<2>(v, red);
  double l0 = 0.0, l1 = 0.0;
  if (det != 0.0) {
    l0 = (n * v[0] - Su * v[1]) / det;
    l1 = (Suu * v[1] - Su * v[0]) / det;
  }
#pragma unroll
  for (int j = 0; j < D_PER; j++) {
    const int i = j * D_THREADS + threadIdx.x;
    double dd = 0.0;
    if (depth_bit(sm, i)) {
      const double u = su[i], r = depth_res(s, t, su, sg, i), q = c + u;
      const double dq = (2.0 * r + er[j]) * s - l0 * (r + u * s) - l1 * s;
      dd = -q * q * dq;
    }
    out[i] = (float)dd;
  }
}

// grad[y, x] = dL/dloss / M * sum over the patches covering (y, x), in patch order; 0 where no patch covers it.  Per
// 256-pixel stretch, warp 0 first lists (in patch order) the patches whose rows meet the stretch's rows, so each pixel
// tests only those few instead of all 64.
__global__ void __launch_bounds__(D_THREADS)
depth_grad_map_kernel(int H, int W, const int64_t* __restrict__ rows, const int64_t* __restrict__ cols,
                      const double* __restrict__ stats, const float* __restrict__ scratch,
                      const float* __restrict__ grad_loss, float* __restrict__ grad) {
  __shared__ int64_t sr[DN], sc[DN];
  __shared__ int list[DN], count;
  for (int k = threadIdx.x; k < DN; k += D_THREADS) {
    sr[k] = rows[k];
    sc[k] = cols[k];
  }
  __syncthreads();
  const double scale = (double)grad_loss[0] * stats[DN * D_STAT];
  const int64_t total = (int64_t)H * W;
  for (int64_t base = (int64_t)blockIdx.x * D_THREADS; base < total; base += (int64_t)gridDim.x * D_THREADS) {
    if (threadIdx.x < 32) {
      const int64_t ya = base / W, yb = (base + D_THREADS - 1 < total ? base + D_THREADS - 1 : total - 1) / W;
      const int lane = threadIdx.x;
      int n = 0;
      for (int k0 = 0; k0 < DN; k0 += 32) {
        const int k = k0 + lane;
        const bool hit = sr[k] <= yb && sr[k] > ya - DP;
        const unsigned b = __ballot_sync(0xffffffffu, hit);
        if (hit) list[n + __popc(b & ((1u << lane) - 1u))] = k;
        n += __popc(b);
      }
      if (lane == 0) count = n;
    }
    __syncthreads();
    const int64_t p = base + threadIdx.x;
    if (p < total) {
      const int64_t y = p / W, x = p % W;
      double sum = 0.0;
      bool covered = false;
      for (int j = 0; j < count; j++) {
        const int k = list[j];
        const int64_t dy = y - sr[k], dx = x - sc[k];
        if ((uint64_t)dy < (uint64_t)DP && (uint64_t)dx < (uint64_t)DP) {
          sum += scratch[(int64_t)k * DPIX + dy * DP + dx];
          covered = true;
        }
      }
      grad[p] = covered ? (float)(sum * scale) : 0.f;
    }
    __syncthreads();      // list and count are rewritten for the next stretch
  }
}

// Per CTA: min and max of q over the masked pixels of its grid-stride share -> part[2 b], part[2 b + 1].
__global__ void __launch_bounds__(D_THREADS)
depth_vis_minmax_kernel(const DepthArgs a, const float* __restrict__ pred, const float* __restrict__ acc,
                        float* __restrict__ part) {
  __shared__ float red[2][D_WARPS];
  float lo = INFINITY, hi = -INFINITY;
  const int64_t total = (int64_t)a.H * a.W;
  for (int64_t p = (int64_t)blockIdx.x * D_THREADS + threadIdx.x; p < total; p += (int64_t)gridDim.x * D_THREADS) {
    const int64_t y = p / a.W, x = p % a.W;
    if (acc[y * a.sa[0] + x * a.sa[1]] > 0.5f) {
      const float q = depth_vis_q(pred[y * a.sp[0] + x * a.sp[1]]);
      lo = depth_min(lo, q);
      hi = depth_max(hi, q);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = depth_min(lo, __shfl_down_sync(0xffffffffu, lo, o));
    hi = depth_max(hi, __shfl_down_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = lo;
    red[1][threadIdx.x >> 5] = hi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < D_WARPS; w++) {
      lo = depth_min(lo, red[0][w]);
      hi = depth_max(hi, red[1][w]);
    }
    part[2 * blockIdx.x] = lo;
    part[2 * blockIdx.x + 1] = hi;
  }
}

// vis[y, x] = (q - lo) / (hi - lo) over the whole (H, W), contiguous.  An empty mask leaves lo = inf, hi = -inf: NaN.
__global__ void __launch_bounds__(D_THREADS)
depth_vis_kernel(const DepthArgs a, const float* __restrict__ pred, const float* __restrict__ part, int parts,
                 float* __restrict__ vis) {
  __shared__ float range[2];
  if (threadIdx.x < 32) {
    float lo = INFINITY, hi = -INFINITY;
    for (int b = threadIdx.x; b < parts; b += 32) {
      lo = depth_min(lo, part[2 * b]);
      hi = depth_max(hi, part[2 * b + 1]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo = depth_min(lo, __shfl_down_sync(0xffffffffu, lo, o));
      hi = depth_max(hi, __shfl_down_sync(0xffffffffu, hi, o));
    }
    if (threadIdx.x == 0) {
      range[0] = lo;
      range[1] = hi;
    }
  }
  __syncthreads();
  const float lo = range[0], den = range[1] - range[0];
  const int64_t total = (int64_t)a.H * a.W;
  for (int64_t p = (int64_t)blockIdx.x * D_THREADS + threadIdx.x; p < total; p += (int64_t)gridDim.x * D_THREADS) {
    const int64_t y = p / a.W, x = p % a.W;
    vis[p] = (depth_vis_q(pred[y * a.sp[0] + x * a.sp[1]]) - lo) / den;
  }
}

static DepthArgs depth_args(int H, int W, int Hd, int Wd, const int64_t* sp, const int64_t* sa, const int64_t* sg) {
  DepthArgs a;
  a.H = H; a.W = W; a.Hd = Hd; a.Wd = Wd;
  for (int k = 0; k < 2; k++) {
    a.sp[k] = sp[k];
    a.sa[k] = sa ? sa[k] : 0;
    a.sg[k] = sg ? sg[k] : 0;
  }
  return a;
}

int launch_depth_loss_fwd(int H, int W, int Hd, int Wd, const float* pred, const int64_t* sp, const float* acc,
                          const int64_t* sa, const float* gt, const int64_t* sg, const int64_t* rows, const int64_t* cols,
                          double* stats, float* loss, cudaStream_t st) {
  const DepthArgs a = depth_args(H, W, Hd, Wd, sp, sa, sg);
  cudaError_t e = cudaFuncSetAttribute(depth_patch_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, D_SMEM);
  if (e != cudaSuccess) return (int)e;
  depth_patch_fwd_kernel<<<DN, D_THREADS, D_SMEM, st>>>(a, pred, acc, gt, rows, cols, stats);
  LGR_CHECK_LAUNCH();
  depth_loss_reduce_kernel<<<1, 32, 0, st>>>(stats, loss);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_depth_loss_bwd(int H, int W, int Hd, int Wd, const float* pred, const int64_t* sp, const float* acc,
                          const int64_t* sa, const float* gt, const int64_t* sg, const int64_t* rows, const int64_t* cols,
                          const double* stats, float* scratch, const float* grad_loss, float* grad, cudaStream_t st) {
  const DepthArgs a = depth_args(H, W, Hd, Wd, sp, sa, sg);
  cudaError_t e = cudaFuncSetAttribute(depth_patch_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, D_SMEM);
  if (e != cudaSuccess) return (int)e;
  depth_patch_bwd_kernel<<<DN, D_THREADS, D_SMEM, st>>>(a, pred, acc, gt, rows, cols, stats, scratch);
  LGR_CHECK_LAUNCH();
  const int64_t blocks = ((int64_t)H * W + D_THREADS - 1) / D_THREADS;
  depth_grad_map_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), D_THREADS, 0, st>>>(H, W, rows, cols, stats, scratch,
                                                                                        grad_loss, grad);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_depth_vis(int H, int W, const float* pred, const int64_t* sp, const float* acc, const int64_t* sa,
                     float* scratch, float* vis, cudaStream_t st) {
  const DepthArgs a = depth_args(H, W, H, W, sp, sa, nullptr);
  const int64_t want = ((int64_t)H * W + 4 * D_THREADS - 1) / (4 * D_THREADS);
  const int parts = (int)(want < LGR_DEPTH_VIS_GRID ? want : LGR_DEPTH_VIS_GRID);
  depth_vis_minmax_kernel<<<parts, D_THREADS, 0, st>>>(a, pred, acc, scratch);
  LGR_CHECK_LAUNCH();
  const int64_t blocks = ((int64_t)H * W + D_THREADS - 1) / D_THREADS;
  depth_vis_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), D_THREADS, 0, st>>>(a, pred, scratch, parts, vis);
  LGR_CHECK_LAUNCH();
  return 0;
}

}  // namespace lgr
