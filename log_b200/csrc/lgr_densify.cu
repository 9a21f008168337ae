// LoG's densification rebuild (Splitter.split_and_remove / split_and_remove_other, LoG/model/splitter.py:138-220) on the
// device.  LoG decides which rows split and which go; this file only rebuilds the tables from the two flags, which LoG
// does on the CPU.  Every table becomes
//     [ rows with ~remove, in index order ]  ++  [ N rows per split parent, parents in ascending index, child c = 0..N-1 ]
// with remove = flag_remove | flag_split when remove_split is set.
//
//   plan      one thread per row: keep / split bits, per-chunk counts and the count of flag_remove; then lgr_prepare.cu's
//             one-CTA scan.  num_keep and S land in the int64 result vector the host reads once, to size the tables.
//   map       lgr_prepare.cu's chunk prefix + ballot rank scatter: map[0, num_keep) the kept rows, map[num_keep, +S) the
//             split parents, both in index order.
//   children  one thread per split parent: log2 N rounds of split_by_uniform in LoG's rounding (explicitly rounded
//             intrinsics, IEEE division and sqrtf, full-precision expf / logf), the N children's xyz and raw scaling, and
//             the statistics LoG prints, reduced per CTA and then in a fixed order.
//   gather    one launch per table: out row r < num_keep copies map[r]; appended row j = r - num_keep takes the parent
//             map[num_keep + j / N] (repeat), the children buffer's row j, or zeros.  A thread moves one 16-, 8-, 4-, 2-
//             or 1-byte unit, the widest that divides the row and both tables' alignment.
// The host runs the gather table by table and swaps each result in, so device memory peaks at the tables before the call
// plus the largest rebuilt table, the children buffer and the row map.
#include "lgr_common.cuh"

namespace lgr {

constexpr int DENS_THREADS = COMPACT_CHUNK;
#ifndef LGR_TREE_GRID
#define LGR_TREE_GRID 528               // 4 CTAs per SM on the 132 SMs of an H100 SXM; grid-stride loops cover any size
#endif
constexpr int DENS_GRID = LGR_TREE_GRID;
static_assert(4 * DENS_GRID <= LGR_DENSIFY_PARTIAL_DOUBLES, "one partial per CTA and statistic");

int launch_compact_scan(int64_t, int32_t*, int64_t*, int64_t*, cudaStream_t);
int launch_compact_scatter(int64_t, const uint8_t*, const int32_t*, const int32_t*, int64_t*, int64_t*, cudaStream_t);

// bits[row]: bit 0 = kept, bit 1 = split parent; two counts per chunk; result[LGR_DENSIFY_REMOVED] += flag_remove rows
__global__ void __launch_bounds__(DENS_THREADS)
densify_plan_kernel(int64_t P, const uint8_t* __restrict__ split, const uint8_t* __restrict__ remove, int remove_split,
                    uint8_t* __restrict__ bits, int32_t* __restrict__ chunk_cnt, int64_t* __restrict__ result) {
  const int64_t nchunks = (P + DENS_THREADS - 1) / DENS_THREADS;
  for (int64_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    const int64_t row = chunk * DENS_THREADS + threadIdx.x;
    int f = 0, r = 0;
    if (row < P) {
      const int s = split[row] != 0;
      r = remove[row] != 0;
      f = !(r || (remove_split && s)) | (s << 1);
      bits[row] = (uint8_t)f;
    }
    const int nk = __syncthreads_count(f & 1), ns = __syncthreads_count(f & 2), nr = __syncthreads_count(r);
    if (threadIdx.x == 0) {
      chunk_cnt[2 * chunk] = nk;
      chunk_cnt[2 * chunk + 1] = ns;
      if (nr) atomicAdd(reinterpret_cast<unsigned long long*>(result + LGR_DENSIFY_REMOVED), (unsigned long long)nr);
    }
  }
}

// split_by_uniform (splitter.py:5-31, 95-130) for one parent, rounded as LoG's torch ops round: build_rotation
// (geometry.py:4-25), argmax of the activated scale (first index on ties), centre + R[:, k] * (+-0.5 s_k), s_k halved,
// and log of the final activated scale on every axis.
template <int N>
__device__ __forceinline__ void split_parent(const float* __restrict__ xyz, const float* __restrict__ scaling,
                                             const float* __restrict__ rotation, int64_t p, float (*c)[3], float* s0,
                                             float* s) {
  const float r = rotation[4 * p], x = rotation[4 * p + 1], y = rotation[4 * p + 2], z = rotation[4 * p + 3];
  const float norm = sqrtf(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r, r), __fmul_rn(x, x)), __fmul_rn(y, y)), __fmul_rn(z, z)));
  const float qr = r / norm, qx = x / norm, qy = y / norm, qz = z / norm;
  float R[3][3];
  R[0][0] = __fadd_rn(1.f, -__fmul_rn(2.f, __fadd_rn(__fmul_rn(qy, qy), __fmul_rn(qz, qz))));
  R[0][1] = __fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qy), -__fmul_rn(qr, qz)));
  R[0][2] = __fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qz), __fmul_rn(qr, qy)));
  R[1][0] = __fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qy), __fmul_rn(qr, qz)));
  R[1][1] = __fadd_rn(1.f, -__fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qx), __fmul_rn(qz, qz))));
  R[1][2] = __fmul_rn(2.f, __fadd_rn(__fmul_rn(qy, qz), -__fmul_rn(qr, qx)));
  R[2][0] = __fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qz), -__fmul_rn(qr, qy)));
  R[2][1] = __fmul_rn(2.f, __fadd_rn(__fmul_rn(qy, qz), __fmul_rn(qr, qx)));
  R[2][2] = __fadd_rn(1.f, -__fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qx), __fmul_rn(qy, qy))));
#pragma unroll
  for (int i = 0; i < 3; i++) { c[0][i] = xyz[3 * p + i]; s0[i] = s[i] = expf(scaling[3 * p + i]); }
  // round n: child a of the previous round becomes children 2a (the -0.5 half) and 2a + 1, written back to front
#pragma unroll
  for (int n = 1; n < N; n *= 2) {
    const int k = (s[1] > s[0]) ? ((s[2] > s[1]) ? 2 : 1) : ((s[2] > s[0]) ? 2 : 0);
    const float h = __fmul_rn(0.5f, s[k]);
#pragma unroll
    for (int a = n - 1; a >= 0; a--) {
#pragma unroll
      for (int i = 0; i < 3; i++) {
        const float d = __fmul_rn(R[i][k], h);
        const float ci = c[a][i];
        c[2 * a][i] = __fadd_rn(ci, -d);
        c[2 * a + 1][i] = __fadd_rn(ci, d);
      }
    }
    s[k] = __fmul_rn(s[k], 0.5f);
  }
}

// children: (N S, 3) xyz, then (N S, 3) raw scaling.  partial[4 blockIdx + q]: this CTA's sums of the parents' activated
// scale, of its per-parent maximum, and of the same two for the children (the four means LoG prints)
template <int N>
__global__ void __launch_bounds__(DENS_THREADS)
densify_children_kernel(int64_t S, const int64_t* __restrict__ parents, const float* __restrict__ xyz,
                        const float* __restrict__ scaling, const float* __restrict__ rotation, float* __restrict__ children,
                        double* __restrict__ partial) {
  __shared__ double red[4][DENS_THREADS / 32];
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int64_t j = (int64_t)blockIdx.x * DENS_THREADS + threadIdx.x; j < S; j += (int64_t)gridDim.x * DENS_THREADS) {
    const int64_t p = parents[j];
    float c[N][3], s0[3], s[3];
    split_parent<N>(xyz, scaling, rotation, p, c, s0, s);
    acc[0] += (double)s0[0] + (double)s0[1] + (double)s0[2];
    acc[1] += (double)fmaxf(fmaxf(s0[0], s0[1]), s0[2]);
    acc[2] += N * ((double)s[0] + (double)s[1] + (double)s[2]);
    acc[3] += N * (double)fmaxf(fmaxf(s[0], s[1]), s[2]);
    const float l0 = logf(s[0]), l1 = logf(s[1]), l2 = logf(s[2]);
    float* cx = children + 3 * N * j;
    float* cs = children + 3 * N * (S + j);
#pragma unroll
    for (int a = 0; a < N; a++) {
      cx[3 * a] = c[a][0]; cx[3 * a + 1] = c[a][1]; cx[3 * a + 2] = c[a][2];
      cs[3 * a] = l0; cs[3 * a + 1] = l1; cs[3 * a + 2] = l2;
    }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < 4; q++) {
    double v = acc[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) red[q][wid] = v;
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double v = 0.0;
    for (int w = 0; w < DENS_THREADS / 32; w++) v += red[threadIdx.x][w];
    partial[4 * blockIdx.x + threadIdx.x] = v;
  }
}

// the four sums over the CTAs in CTA order, as means, into the result vector's doubles
__global__ void densify_stats_kernel(int64_t S, int N, int ctas, const double* __restrict__ partial, int64_t* __restrict__ result) {
  const int q = threadIdx.x;
  if (q >= 4) return;
  double v = 0.0;
  for (int b = 0; b < ctas; b++) v += partial[4 * b + q];
  const double count[4] = {3.0 * S, (double)S, 3.0 * N * S, (double)N * S};
  reinterpret_cast<double*>(result + LGR_DENSIFY_STATS)[q] = v / count[q];
}

template <class T>
__global__ void __launch_bounds__(DENS_THREADS)
densify_gather_kernel(int64_t num_keep, int64_t rows_out, int N, int units, int mode, const int64_t* __restrict__ map,
                      const T* __restrict__ src, const T* __restrict__ appended, T* __restrict__ dst) {
  const int64_t total = rows_out * units;
  const bool narrow = total <= 0xffffffffLL;            // 32-bit division where the index allows it
  for (int64_t i = (int64_t)blockIdx.x * DENS_THREADS + threadIdx.x; i < total; i += (int64_t)gridDim.x * DENS_THREADS) {
    const int64_t r = narrow ? (int64_t)((uint32_t)i / (uint32_t)units) : i / units;
    const int u = (int)(i - r * units);
    T v;
    if (r < num_keep) v = src[map[r] * units + u];
    else if (mode == LGR_DENSIFY_REPEAT) v = src[map[num_keep + (r - num_keep) / N] * units + u];
    else if (mode == LGR_DENSIFY_CHILDREN) v = appended[(r - num_keep) * units + u];
    else v = T{};
    dst[i] = v;
  }
}

int launch_densify_plan(int64_t P, const uint8_t* split, const uint8_t* remove, int remove_split, int32_t* scratch,
                        int64_t* result, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(result, 0, LGR_DENSIFY_RESULTS * sizeof(int64_t), st);
  if (e != cudaSuccess) return (int)e;
  int32_t* chunk_cnt = scratch;
  uint8_t* bits = reinterpret_cast<uint8_t*>(scratch + 2 * ((P + DENS_THREADS - 1) / DENS_THREADS) + 2);
  if (P > 0) {
    densify_plan_kernel<<<DENS_GRID, DENS_THREADS, 0, st>>>(P, split, remove, remove_split, bits, chunk_cnt, result);
    LGR_CHECK_LAUNCH();
  }
  return launch_compact_scan(P, chunk_cnt, result + LGR_DENSIFY_KEEP, result + LGR_DENSIFY_SPLIT, st);
}

int launch_densify_map(int64_t P, int64_t num_keep, const int32_t* scratch, int64_t* map, cudaStream_t st) {
  if (P == 0) return 0;
  const uint8_t* bits = reinterpret_cast<const uint8_t*>(scratch + 2 * ((P + DENS_THREADS - 1) / DENS_THREADS) + 2);
  return launch_compact_scatter(P, bits, scratch, nullptr, map, map + num_keep, st);
}

int launch_densify_children(int64_t S, int N, const int64_t* parents, const float* xyz, const float* scaling,
                            const float* rotation, float* children, double* partial, int64_t* result, cudaStream_t st) {
  if (S == 0) return 0;
  if (N == 2) densify_children_kernel<2><<<DENS_GRID, DENS_THREADS, 0, st>>>(S, parents, xyz, scaling, rotation, children, partial);
  else if (N == 4) densify_children_kernel<4><<<DENS_GRID, DENS_THREADS, 0, st>>>(S, parents, xyz, scaling, rotation, children, partial);
  else densify_children_kernel<8><<<DENS_GRID, DENS_THREADS, 0, st>>>(S, parents, xyz, scaling, rotation, children, partial);
  LGR_CHECK_LAUNCH();
  densify_stats_kernel<<<1, 32, 0, st>>>(S, N, DENS_GRID, partial, result);
  LGR_CHECK_LAUNCH();
  return 0;
}

template <class T>
static int gather_as(int64_t num_keep, int64_t rows_out, int N, int64_t row_bytes, int mode, const int64_t* map, const void* src,
                     const void* appended, void* dst, cudaStream_t st) {
  densify_gather_kernel<T><<<DENS_GRID, DENS_THREADS, 0, st>>>(num_keep, rows_out, N, (int)(row_bytes / sizeof(T)), mode, map,
                                                              static_cast<const T*>(src), static_cast<const T*>(appended),
                                                              static_cast<T*>(dst));
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_densify_gather(int64_t num_keep, int64_t rows_out, int N, int64_t row_bytes, int mode, const int64_t* map,
                          const void* src, const void* appended, void* dst, cudaStream_t st) {
  if (rows_out == 0) return 0;
  uintptr_t align = (uintptr_t)src | (uintptr_t)dst | (uintptr_t)appended | (uintptr_t)row_bytes;
  if (align % 16 == 0) return gather_as<int4>(num_keep, rows_out, N, row_bytes, mode, map, src, appended, dst, st);
  if (align % 8 == 0) return gather_as<long long>(num_keep, rows_out, N, row_bytes, mode, map, src, appended, dst, st);
  if (align % 4 == 0) return gather_as<int32_t>(num_keep, rows_out, N, row_bytes, mode, map, src, appended, dst, st);
  if (align % 2 == 0) return gather_as<int16_t>(num_keep, rows_out, N, row_bytes, mode, map, src, appended, dst, st);
  return gather_as<int8_t>(num_keep, rows_out, N, row_bytes, mode, map, src, appended, dst, st);
}

}  // namespace lgr
